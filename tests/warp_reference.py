"""Float64 reference of the warp side: the 8-NN search (df_knn8, csrc/warp.cu, warp_common.cuh), the dual-quaternion blend warp (df_warp) and
per-voxel warped fusion (df_integrate_warped, csrc/fusion.cu), with the search path the fusion kernel takes.  numpy and scipy, no oracle
call: it restates the operations, not the float32 order of either implementation, so an operation both get wrong in the same way fails here.

Every float32 input (node vertices, quaternions and weights, voxel size, truncation distance, intrinsics, poses, query points) is taken at
its float32 value and then computed on exactly in float64.  U = 2^-24 is the unit roundoff of float32: one rounding of a value a errs by at
most U |a|.  Bars are first order (products of two error terms are dropped); each states the roundings of the float32 chain it covers.

k-NN (knn64).  The kernels' squared distance d0*d0 + d1*d1 + d2*d2 (di = q_i - v_i) carries one rounding per difference (2U relative on
the square), one per square and one per sum: it is within 5U d^2 of the exact value; the margin taken is m = 6U d^2.  When the query itself
is a float32 value within delta (per axis) of the exact point (the fusion kernel's voxel position), the exact distance moves by at most
2 |x - v| |delta| + |delta|^2 more.  A distance whose every float32 step is exact (each difference, square and partial sum representable,
so that any order of the sum gives it) has no margin: nodes on the voxel lattice then tie exactly on both sides and both rank by index.  The
kernel returns the 8 smallest by (float distance, index): a set S is admissible when max_{i in S} (d_i - m_i) <= min_{j not in S} (d_j + m_j),
and the query is ambiguous when the exact 8-set is not forced (some member's upper end reaches a non-member's lower end).

Warp (warp64).  w_i = exp(-d_i^2 / (2 s_i^2)) (s_i the node weight).  The kernel's argument carries 2U relative (2 s s and the division)
plus the distance margin over 2 s^2; the double exp narrowed to float adds U w: dw_i = w_i (2U a_i + m_i / (2 s_i^2) + 1.5U), a_i the exact
argument.  t_i = 2 dual_i conj(r_i / |r_i|) (DualQuaternion::getTranslation) is formed in float32 within 8U (|2 dual_i| x |r_i / |r_i||)_k
in component k, the quaternion product taken over the magnitudes of the factors (3U of normalisation, 4U of products and sums): a component
whose terms are all exact zeros (no rotation, a pure translation) carries no error.
The blend sums R = sum w_i r_i and T = sum w_i t_i (8 products and 8 sums: 9U sum |w_i x_i| per component), normalises R to r and applies
DualQuaternion(T, r).transform: the translation it adds is T |r| = T (up to 12U |T|_1 for the two quaternion products and the renormalised
rotation in between), the rotation is R(r) x.  The direction of r moves by eta = 2 |dR|_2 / |R| + 4U, and R(r) x by 4 eta |x| + 12U |x| (the
rotation matrix of a unit quaternion is 4-Lipschitz; qrotate's cross products and its own normalisation).  Where every neighbour's rotation
is exactly (1, 0, 0, 0) the rotation is exact in float32 and only the translation terms remain: x + T, one more rounding.  The blend is
conditioned on |R| / sum w_i: below COND_MIN (antipodal cancellation) the point is ambiguous.  warp_to_live (A, b) is applied last: the bar
goes through |A| and the product adds 4U (|A| |p| + |b|).  Normals: the full transform (rotation and T, as the reference also translates
normals), or DF_WARP_NORMAL_ROTATE_ONLY: R(r) n, then A n.

Warped fusion (integrate_warped64).  A voxel (x, y, z) sits at P = (x vsx, y vsy, z vsz), world position x_c = R P + t exactly; the kernel
forms it with one aff_mul (the three products x vsx .. and the affine map: <= 5U (sum_j |R_ij P_j| + |t_i|) per coordinate, 0 where every
float32 step is exact), and searches, warps and projects that float32 point.  Then x_t = W x_w + w (world2cam, 4U as above),
u = fx X / Z + cx moves by du = |fx| (e_x + |X / Z| e_z) / Z + U |fx X / Z| + U |u|, v likewise; the pixel (int)u after the tests u >= 0,
u < cols is floor(u) in [0, cols), a decision with integer thresholds: a voxel whose u lies within du of an integer has two candidate
columns (four candidate pixels at most).  tz > 0 is ambiguous within e_z.  rho = Dp - Z with Dp = mm 0.001 (the constant 0.001f and the
product: 2U |Dp|, the difference U |rho|): the gate rho > -trunc is ambiguous within drho.  The quantised weight clamp(rint(w scale), 1,
max_weight), w = sum_valid sqrt(d_i^2) / 8 (sum / 8 also when fewer than 8 nodes exist): each root moves by min(m / d, sqrt(m)) + U d, the
sum by 9U sum d, the product with scale by U; a weight whose interval holds a rounding boundary of rint (near .5) has two candidates.
The update F' = (F W + tsdf wq) / (W + wq), tsdf = min(1, rho / trunc), is checked as tsdf_reference checks the rigid one: tsdf errs by
drho / trunc + 2U |tsdf|, the product tsdf wq, the fma and the division by one rounding each, so before the rounding to half the float32
value is within e = (dtsdf wq + U |tsdf wq| + U |F W + tsdf wq|) / (W + wq) + U |F'| of F', and the stored half within
bar = halfulp(|F'| + e) + e; W' = min(W + wq, max_weight) exactly.  A voxel is ambiguous only when its candidates (pixels x gate x weight
outcomes) lead to different stored words, or when its neighbour set is not forced, its blend is ill-conditioned or its projection moves by
a quarter pixel or more ('wild': any update with |F| <= 1 and a weight in range, or none).

Search path (search_path).  Restates from csrc/fusion.cu which search each block and each 8 x 4 x 8 voxel run of the fusion kernel takes,
in float64: a block (32 x 8 x zchunk voxels) lists the nodes within (d8(cb) + 2 h_b) (1.0002) of its centre cb and uses the list when it
holds 8 to FUS_BLOCK_CAP nodes; a run of a listed block lists those within (d8(c) + 2 h) (1.0002) of its centre c and ranks them when it
holds at most FUS_LIST_CAP, else it walks the BVH; M < 8 or M > 8192 (no BVH) use no lists, and without a BVH every voxel walks the grid.
The kernel's d8 is the 8th smallest of 32 or 64 lane minima (>= the exact d8), so its counts are at least these: the cases are built so
that the outcome holds by a wide margin, and the restatement is approximate on purpose."""
from __future__ import annotations

import itertools

import numpy as np
from scipy.spatial import cKDTree

from tsdf_reference import halfulp, halves  # noqa: F401  (halves re-exported for the tests)

U = 2.0 ** -24
KNN_MARGIN = 6.0                  # distance margin, in units of U d^2
COND_MIN = 0.5                    # |sum w_i r_i| / sum w_i below this: the blend is ill-conditioned, the point is ambiguous
MAX_TIE_SETS = 70                 # admissible neighbour sets enumerated per ambiguous voxel before it is taken as wild (C(8, 4))


def f64(a):
    """float32 values (the kernels' parameters) in float64"""
    return np.asarray(a, np.float32).astype(np.float64)


# ------------------------------------------------------------------ quaternions --------------------------------------------------------------
def qmul(a, b):
    aw, ax, ay, az = np.moveaxis(a, -1, 0)
    bw, bx, by, bz = np.moveaxis(b, -1, 0)
    return np.stack([aw * bw - ax * bx - ay * by - az * bz, aw * bx + ax * bw + ay * bz - az * by,
                     aw * by - ax * bz + ay * bw + az * bx, aw * bz + ax * by - ay * bx + az * bw], -1)


def qmul_abs(a, b):
    """the quaternion product's terms summed over magnitudes, per component: a bound on the rounding of each component of qmul(a, b)"""
    aw, ax, ay, az = np.moveaxis(np.abs(a), -1, 0)
    bw, bx, by, bz = np.moveaxis(np.abs(b), -1, 0)
    return np.stack([aw * bw + ax * bx + ay * by + az * bz, aw * bx + ax * bw + ay * bz + az * by,
                     aw * by + ax * bz + ay * bw + az * bx, aw * bz + ax * by + ay * bx + az * bw], -1)


def conj(q):
    return q * np.array([1.0, -1.0, -1.0, -1.0])


def rotate(q, v):
    """R(q / |q|) v"""
    q = q / np.linalg.norm(q, axis=-1, keepdims=True)
    p = np.concatenate([np.zeros(v.shape[:-1] + (1,)), v], -1)
    return qmul(qmul(q, p), conj(q))[..., 1:]


def node_translations(nodes):
    """t_i = 2 dual_i conj(r_i / |r_i|): [M, 4]"""
    n = f64(nodes)
    r = n[:, 3:7] / np.linalg.norm(n[:, 3:7], axis=1, keepdims=True)
    return qmul(2.0 * n[:, 7:11], conj(r))


# ------------------------------------------------------------------ k-NN ---------------------------------------------------------------------
def _f32_exact_dist(q, v):
    """True where every float32 step of |q - v|^2 is exact (q [n, 3], v [n, k, 3] float32 values in float64)"""
    d = q[:, None, :] - v
    ok = (d.astype(np.float32).astype(np.float64) == d).all(-1)
    s = d * d
    ok &= (s.astype(np.float32).astype(np.float64) == s).all(-1)
    for a, b in ((0, 1), (0, 2), (1, 2)):
        p = s[..., a] + s[..., b]
        ok &= p.astype(np.float32).astype(np.float64) == p
    t = s.sum(-1)
    return ok & (t.astype(np.float32).astype(np.float64) == t)


def _margins(q, v, d2, delta, q_exact):
    m = KNN_MARGIN * U * d2 + 2.0 * np.sqrt(d2) * delta[:, None] + delta[:, None] ** 2
    ex = _f32_exact_dist(q, v) & q_exact[:, None]
    return np.where(ex, 0.0, m)


def knn64(nodes, queries, delta=None, q_exact=None, kmax=24):
    """the exact 8-NN of float64 queries [n, 3] among the node vertices.  delta [n]: |error| of the float32 query the kernel searches from
    (0: the query is exact); q_exact [n]: the float32 query equals the exact one.  Returns a dict: idx [n, 8] (-1 past M), d2 [n, 8] (exact),
    m [n, 8] (margins), forced [n], and for each query the candidates the admissibility test needs: cand_idx, cand_d2, cand_m [n, k]
    (k nearest, sorted by (distance, index); np.inf padded)"""
    V = f64(nodes)[:, :3]
    M = len(V)
    q = np.asarray(queries, np.float64)
    n = len(q)
    delta = np.zeros(n) if delta is None else np.asarray(delta, np.float64)
    q_exact = np.ones(n, bool) if q_exact is None else np.asarray(q_exact, bool)
    k = min(M, kmax)
    tree = cKDTree(V)
    _, ci = tree.query(q, k=k)
    ci = ci.reshape(n, k)
    vv = V[ci]
    d2 = ((q[:, None, :] - vv) ** 2).sum(-1)
    # rank by (exact distance, index): sort by index, then stably by distance
    key = np.argsort(ci, axis=1, kind="stable")
    ci, d2, vv = np.take_along_axis(ci, key, 1), np.take_along_axis(d2, key, 1), np.take_along_axis(vv, key[..., None], 1)
    key = np.argsort(d2, axis=1, kind="stable")
    ci, d2, vv = np.take_along_axis(ci, key, 1), np.take_along_axis(d2, key, 1), np.take_along_axis(vv, key[..., None], 1)
    m = _margins(q, vv, d2, delta, q_exact)
    if k < M:
        # the k-th candidate must be beyond reach of the 8th: else search wider for those queries (all nodes)
        lim = (d2[:, :8] + m[:, :8]).max(1)
        wide = np.flatnonzero(d2[:, -1] - m[:, -1] <= lim)
        if len(wide):
            ca = np.broadcast_to(np.arange(M), (len(wide), M))
            vw = V[ca]
            dw = ((q[wide, None, :] - vw) ** 2).sum(-1)
            key = np.argsort(dw, axis=1, kind="stable")
            ca, dw, vw = np.take_along_axis(ca, key, 1), np.take_along_axis(dw, key, 1), np.take_along_axis(vw, key[..., None], 1)
            mw = _margins(q[wide], vw, dw, delta[wide], q_exact[wide])
            # keep every candidate up to the last one still within reach of the 8th: the rest is out of reach for certain
            reach = dw - mw <= (dw[:, :8] + mw[:, :8]).max(1)[:, None]
            kk = int(min(M, max(k, np.where(reach, np.arange(M), 0).max() + 2)))
            full = np.full((n, kk), np.inf)
            ci2 = np.full((n, kk), -1, np.int64)
            for arr, src in ((full, d2), (ci2, ci)):
                arr[:, :k] = src
            m2 = np.full((n, kk), np.inf)
            m2[:, :k] = m
            ci2[wide], full[wide], m2[wide] = ca[:, :kk], dw[:, :kk], mw[:, :kk]
            ci, d2, m = ci2, full, m2
    idx = np.full((n, 8), -1, np.int64)
    dd = np.full((n, 8), np.inf)
    mm = np.zeros((n, 8))
    j = min(8, M)
    idx[:, :j], dd[:, :j], mm[:, :j] = ci[:, :j], d2[:, :j], m[:, :j]
    # a node at the same vertex as a member (duplicated vertices) has the same float distance and a higher index: it never displaces it
    _, first = np.unique(V, axis=0, return_inverse=True)
    cv = np.where(ci >= 0, first.reshape(-1)[np.where(ci >= 0, ci, 0)], -1 - np.arange(ci.shape[1]))     # vertex class of each candidate
    if ci.shape[1] > 8:
        # member i (of the first 8) beats non-member j for certain: its interval lies below j's, or both distances are exact in float32
        # (then both rank by (distance, index) as here), or j is i's twin
        di, mi, dj, mj = d2[:, :8, None], m[:, :8, None], d2[:, None, 8:], m[:, None, 8:]
        beat = (di + mi < dj - mj) | ((mi == 0) & (mj == 0)) | (cv[:, :8, None] == cv[:, None, 8:]) | ~np.isfinite(dj)
        forced = beat.all((1, 2))
    else:
        forced = np.ones(n, bool)
    return {"idx": idx, "d2": dd, "m": mm, "forced": forced, "cand_idx": ci, "cand_d2": d2, "cand_m": m, "cand_v": cv}


def knn_admissible(ref, idx):
    """True per query where the set idx [n, 8] (-1 past M) is one the kernel may return"""
    ci, d2, m = ref["cand_idx"], ref["cand_d2"], ref["cand_m"]
    n = len(idx)
    M_valid = (ref["idx"] >= 0).sum(1)
    got = np.sort(np.where(idx >= 0, idx, np.iinfo(np.int64).max), 1)
    ok = ((idx >= 0).sum(1) == M_valid)
    member = (ci[:, :, None] == got[:, None, :]).any(-1) & (ci >= 0)
    # no non-member j may beat a member i for certain: j's interval below i's, or both exact (or twins, which tie exactly in float32
    # too) with j first in (distance, index) order
    cv = ref["cand_v"]
    di, mi, ii = d2[:, :, None], m[:, :, None], ci[:, :, None]
    dj, mj, ij = d2[:, None, :], m[:, None, :], ci[:, None, :]
    exact = ((mi == 0) & (mj == 0)) | (cv[:, :, None] == cv[:, None, :])
    first = (dj < di) | ((dj == di) & (ij < ii))
    beaten = (dj + mj < di - mi) | (exact & first)
    ok &= ~(beaten & member[:, :, None] & (~member & (ci >= 0))[:, None, :]).any((1, 2))
    return ok & (member.sum(1) == M_valid)            # every returned index is among the candidates


def admissible_sets(ref, i):
    """the neighbour sets the kernel may return for query i (sorted index tuples), or None when there are more than MAX_TIE_SETS"""
    ci, d2, m = ref["cand_idx"][i], ref["cand_d2"][i], ref["cand_m"][i]
    ok = ci >= 0
    ci, d2, m = ci[ok], d2[ok], m[ok]
    if len(ci) <= 8:
        return [tuple(sorted(ci))]
    hi8 = (d2[:8] + m[:8]).max()
    sure = d2 + m < (d2[8:] - m[8:]).min()
    group = np.flatnonzero(~sure & (d2 - m <= hi8))
    need = 8 - int(sure.sum())
    if need <= 0 or len(group) > 16:
        return None
    combos = []
    for comb in itertools.combinations(group, need):
        members = np.concatenate([np.flatnonzero(sure), np.asarray(comb, np.int64)])
        inside = np.zeros(len(ci), bool)
        inside[members] = True
        if (d2[inside] - m[inside]).max() <= (d2[~inside] + m[~inside]).min():
            combos.append(tuple(sorted(ci[inside])))
        if len(combos) > MAX_TIE_SETS:
            return None
    return combos


# ------------------------------------------------------------------ warp ---------------------------------------------------------------------
def blend64(nodes, x, idx, d2, m, delta=None, perturb=None):
    """the DQB warp of points x [n, 3] by the neighbours idx [n, 8] (-1: none) at exact squared distances d2 with margins m.  delta [n]:
    |error| of the float32 point the kernel transforms.  Returns (rotation quaternion r [n, 4] (unit), T [n, 4], point [n, 3], its bar [n, 3],
    rotation bar factor erot_rel [n] (the rotation's error per unit length of the rotated vector), translation bar eT [n, 3], ill-conditioned
    [n], identity [n])"""
    n_ = f64(nodes)
    x = np.asarray(x, np.float64)
    n = len(x)
    delta = np.zeros(n) if delta is None else delta
    valid = idx >= 0
    if perturb == "k7":
        valid = valid & (np.arange(8) < 7)
    ii = np.where(valid, idx, 0)
    sig = n_[ii, 11]
    a = np.where(valid, d2 / (2 * sig * sig), 0.0)
    w = np.where(valid, np.exp(-2 * a if perturb == "exp_no_half" else -a), 0.0)
    dw = np.where(valid, w * (2 * U * a + np.where(valid, m, 0.0) / (2 * sig * sig) + 1.5 * U), 0.0)
    r = n_[ii, 3:7]
    t = node_translations(nodes)[ii] if perturb != "no_conj" else 2.0 * n_[ii, 7:11]
    rn = np.abs(r) / np.linalg.norm(r, axis=-1, keepdims=True)
    et = 8 * U * qmul_abs(np.abs(2.0 * n_[ii, 7:11]), rn)               # per component: the product's terms over magnitudes
    R = (w[..., None] * r).sum(1)
    T = (w[..., None] * t).sum(1)
    rmax = np.abs(r).max(-1)
    dR = ((dw + 9 * U * w) * rmax).sum(1)
    dT = (dw[..., None] * np.abs(t) + w[..., None] * et + 9 * U * w[..., None] * np.abs(t)).sum(1)     # [n, 4]
    Rn = np.linalg.norm(R, axis=1)
    W = w.sum(1)
    with np.errstate(invalid="ignore", divide="ignore"):
        ill = ~(Rn >= COND_MIN * W)
        rq = R / Rn[:, None]
    ident = ((r == np.array([1.0, 0, 0, 0])).all(-1) | ~valid).all(1)
    with np.errstate(invalid="ignore", divide="ignore"):
        eta = 2 * 2 * dR / Rn + 4 * U
    erot_rel = np.where(ident, 0.0, 4 * eta + 12 * U)
    eTr = dT[:, 1:] + np.where(ident, 0.0, 12 * U * np.abs(T).sum(1))[:, None]
    rx = np.where(ident[:, None], x, rotate(np.where(ill[:, None], np.array([1.0, 0, 0, 0]), rq), x))
    p = rx + T[:, 1:]
    xn = np.linalg.norm(x, axis=1)
    bar = (erot_rel * xn)[:, None] + eTr + delta[:, None] + U * (np.abs(rx) + np.abs(T[:, 1:])) * np.where(ident, 0.0, 1.0)[:, None] \
        + U * np.abs(p)
    return rq, T, p, bar, erot_rel, eTr, ill, ident


def affine64(A, p, bar, translate=True):
    """(A p + b, bar) of a float32 affine map (R, t) applied in float32 to points within bar of p"""
    R, b = f64(A[0]).reshape(3, 3), f64(A[1]).reshape(3)
    out = p @ R.T + (b if translate else 0.0)
    ob = bar @ np.abs(R).T + 4 * U * (np.abs(p) @ np.abs(R).T + (np.abs(b) if translate else 0.0))
    return out, ob


def warp64(nodes, points, normals, w2l, rotate_only=False, idx=None, perturb=None):
    """df_warp of float32 points and normals [n, 3]: (points, point bars, normals, normal bars, ambiguous [n], knn reference).  idx [n, 8]:
    evaluate with these neighbour sets (the kernel's own where the float64 set is not forced) instead of the exact ones"""
    x = f64(points)[:, :3]
    nr = f64(normals)[:, :3]
    if perturb == "w2l_first":                        # warp_to_live applied before the blend instead of after it
        x = x @ f64(w2l[0]).reshape(3, 3).T + f64(w2l[1]).reshape(3)
        nr = nr @ f64(w2l[0]).reshape(3, 3).T
        w2l = (np.eye(3), np.zeros(3))
    ref = knn64(nodes, x)
    use = ref["idx"] if idx is None else np.asarray(idx, np.int64)
    V = f64(nodes)[:, :3]
    d2 = np.where(use >= 0, ((x[:, None, :] - V[np.where(use >= 0, use, 0)]) ** 2).sum(-1), np.inf)
    m = KNN_MARGIN * U * np.where(use >= 0, d2, 0.0)
    rq, T, p, pbar, erot_rel, eTr, ill, ident = blend64(nodes, x, use, d2, m, perturb=perturb)
    nn = np.where(ident[:, None], nr, rotate(np.where(ill[:, None], np.array([1.0, 0, 0, 0]), rq), nr))
    nmag = np.linalg.norm(nr, axis=1)
    if rotate_only:
        nbar = (erot_rel * nmag)[:, None] + U * np.abs(nn) + np.where(ident, 0.0, 3 * U * nmag)[:, None]
        n_out, nb_out = affine64(w2l, nn, nbar, translate=False)
    else:
        nn = nn + T[:, 1:]
        nbar = (erot_rel * nmag)[:, None] + eTr + U * np.abs(nn) + np.where(ident, 0.0, 3 * U * nmag)[:, None]
        n_out, nb_out = affine64(w2l, nn, nbar)
    p_out, pb_out = affine64(w2l, p, pbar)
    amb = ill | (~ref["forced"] if idx is None else np.zeros(len(x), bool))
    return p_out, pb_out, n_out, nb_out, amb, ref


def warp_check(got_p, got_n, ref, sel=None):
    """(violations, worst point ratio, worst normal ratio, checked) of the kernel's points and normals [n, >= 3] against warp64's result"""
    p, pb, nn, nb, amb = ref[:5]
    ok = ~amb if sel is None else (~amb & sel)
    rp = np.abs(f64(got_p)[ok, :3] - p[ok]) / pb[ok]
    rn = np.abs(f64(got_n)[ok, :3] - nn[ok]) / nb[ok]
    bad = int(np.count_nonzero(~(rp <= 1.0)) + np.count_nonzero(~(rn <= 1.0)))
    return bad, float(rp.max()) if rp.size else 0.0, float(rn.max()) if rn.size else 0.0, int(ok.sum())


# ------------------------------------------------------------------ warped fusion ------------------------------------------------------------
def voxel_positions(dims, vs, vol2world, lin=None, perturb=None):
    """(P [n, 3] exact volume-frame positions, x_c [n, 3] world, delta [n] (norm of the per-axis bound), exact [n]) of the voxels with flat
    (z, y, x) indices lin (all when None)"""
    Dx, Dy, Dz = (int(d) for d in dims)
    lin = np.arange(Dx * Dy * Dz) if lin is None else np.asarray(lin, np.int64)
    x, y, z = lin % Dx, (lin // Dx) % Dy, lin // (Dx * Dy)
    vs = f64(vs)
    if perturb == "swap_vsy_vsz":
        vs = vs[[0, 2, 1]]
    R, t = f64(vol2world[0]).reshape(3, 3), f64(vol2world[1]).reshape(3)
    P = np.stack([x * vs[0], y * vs[1], z * vs[2]], 1)
    if perturb == "half_voxel":
        P = P + 0.5 * vs
    xc = P @ R.T + t
    e = 5 * U * (np.abs(P) @ np.abs(R).T + np.abs(t))
    # a position whose every float32 step is exact (the three products, the nine products and the partial sums left to right)
    ex = (P.astype(np.float32).astype(np.float64) == P).all(1)
    acc = np.zeros_like(P)
    for j in range(3):
        prod = P[:, j:j + 1] * R[:, j][None, :]
        ex &= (prod.astype(np.float32).astype(np.float64) == prod).all(1)
        acc = acc + prod
        ex &= (acc.astype(np.float32).astype(np.float64) == acc).all(1)
    acc = acc + t
    ex &= (acc.astype(np.float32).astype(np.float64) == acc).all(1)
    e[ex] = 0.0
    return P, xc, np.linalg.norm(e, axis=1), ex


def warp_voxels(nodes, dims, vs, vol2world, lin=None, perturb=None):
    """the field's part of warped fusion, which does not depend on the frame: the voxels' k-NN, their warped world positions and bars.  A
    dict: lin, x_w [n, 3], bar [n, 3], sqrt sums (sd [n], dsd [n]: sum_valid sqrt(d^2) and its error), forced [n], ill [n], alt (for
    voxels whose neighbour set is not forced: a list of (x_w, bar, sd, dsd) per admissible set, or None)"""
    P, xc, delta, ex = voxel_positions(dims, vs, vol2world, lin, perturb)
    ref = knn64(nodes, xc, delta, ex)
    lin = np.arange(len(xc)) if lin is None else np.asarray(lin, np.int64)

    def evaluate(rows, idx):
        V = f64(nodes)[:, :3]
        valid = idx >= 0
        d2 = np.where(valid, ((xc[rows, None, :] - V[np.where(valid, idx, 0)]) ** 2).sum(-1), 0.0)
        m = np.where(valid, _margins(xc[rows], V[np.where(valid, idx, 0)], d2, delta[rows], ex[rows]), 0.0)
        _, _, p, bar, _, _, ill, _ = blend64(nodes, xc[rows], idx, d2, m, delta[rows], perturb)
        d = np.sqrt(d2)
        sd = np.where(valid, d, 0.0).sum(1)
        if perturb == "mean_weight":                  # the mean over the valid neighbours instead of sum / 8
            sd = sd * 8 / np.maximum(valid.sum(1), 1)
        with np.errstate(divide="ignore", invalid="ignore"):
            droot = np.where(valid, np.minimum(np.where(d > 0, m / np.maximum(d, 1e-300), np.inf), np.sqrt(m)) + U * d, 0.0)
        dsd = droot.sum(1) + 9 * U * sd
        return p, bar, sd, dsd, ill

    rows = np.arange(len(xc))
    p, bar, sd, dsd, ill = evaluate(rows, ref["idx"])
    alt = {}
    for i in np.flatnonzero(~ref["forced"]):
        sets = admissible_sets(ref, i)
        if sets is None:
            alt[i] = None
            continue
        ids = np.full((len(sets), 8), -1, np.int64)
        for s, st in enumerate(sets):
            ids[s, :len(st)] = st
        alt[i] = evaluate(np.full(len(sets), i), ids)
    return {"lin": lin, "x_w": p, "bar": bar, "sd": sd, "dsd": dsd, "forced": ref["forced"], "ill": ill, "alt": alt, "idx": ref["idx"]}


def _frame_outcomes(xw, bar, sd, dsd, F0, W0, depth, K, world2cam, trunc, max_w, weight_scale):
    """per voxel row: the candidate outcomes of one frame.  Returns (may [c, n], must [c, n], new [c, n], cbar [c, n], wq [c, n],
    wild [n]) over c = 4 pixels x 2 weights"""
    fx, fy, cx, cy = f64(K)
    rows, cols = depth.shape
    trunc = float(np.float32(trunc))
    xt, et = affine64(world2cam, xw, bar)
    X, Y, Z = xt.T
    ex, ey, ez = et.T
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        qx, qy = X / Z, Y / Z
        u, v = fx * qx + cx, fy * qy + cy
        du = abs(fx) * (ex + np.abs(qx) * ez) / np.abs(Z) + U * np.abs(fx * qx) + U * np.abs(u)
        dv = abs(fy) * (ey + np.abs(qy) * ez) / np.abs(Z) + U * np.abs(fy * qy) + U * np.abs(v)
        off = (u + du < 0) | (u - du >= cols) | (v + dv < 0) | (v - dv >= rows)
    front, maybe = Z > ez, Z > -ez
    wild = maybe & ~off & ~((du < 0.25) & (dv < 0.25))
    sane = maybe & ~wild & ~off
    n = len(X)
    ul, uh, vl, vh = (np.full(n, -1, np.int64) for _ in range(4))
    ul[sane], uh[sane] = np.floor(u[sane] - du[sane]), np.floor(u[sane] + du[sane])
    vl[sane], vh[sane] = np.floor(v[sane] - dv[sane]), np.floor(v[sane] + dv[sane])
    # the quantised weight's candidates
    if weight_scale > 0:
        s = float(np.float32(weight_scale))
        ws = sd / 8 * s
        dws = dsd / 8 * s + U * ws
        wqs = [np.clip(np.rint(ws - dws), 1, max_w), np.clip(np.rint(ws + dws), 1, max_w)]
    else:
        wqs = [np.ones(n), np.ones(n)]
    D = depth.astype(np.float64)
    may, must, new, cbar, wq_out = [], [], [], [], []
    for cu, cv in ((ul, vl), (uh, vl), (ul, vh), (uh, vh)):
        ok = sane & (cu >= 0) & (cu < cols) & (cv >= 0) & (cv < rows)
        Dp = np.zeros(n)
        Dp[ok] = D[cv[ok], cu[ok]] * 1e-3
        live = ok & (Dp != 0)
        rho = Dp - Z
        drho = ez + 2 * U * np.abs(Dp) + U * np.abs(rho)
        mu = live & front & (rho > -trunc + drho)
        ma = live & maybe & (rho > -trunc - drho)
        tsdf = np.minimum(1.0, rho / trunc)
        dts = np.where(rho / trunc > 1.0 + drho / trunc + 4 * U, 0.0, drho / trunc + 2 * U * np.abs(tsdf))
        for wq in wqs:
            nv = (F0 * W0 + tsdf * wq) / (W0 + wq)
            e = (dts * wq + U * np.abs(tsdf * wq) + U * np.abs(F0 * W0 + tsdf * wq)) / (W0 + wq) + U * np.abs(nv)
            may.append(ma); must.append(mu); new.append(np.where(ma, nv, np.nan)); cbar.append(halfulp(np.abs(nv) + e) + e); wq_out.append(wq)
    return np.stack(may), np.stack(must), np.stack(new), np.stack(cbar), np.stack(wq_out), wild


def integrate_warped64(prev, warped, depth, K, world2cam, trunc, max_w, weight_scale):
    """one frame's update of the volume words prev (flat, (z, y, x) order) on the voxels warp_voxels evaluated.  Returns a dict as
    tsdf_reference.integrate64's: upd, amb (over those voxels), new, bar, w_new, and the candidates of the ambiguous voxels"""
    lin = warped["lin"]
    F0, W0 = halves(np.asarray(prev, np.uint32)[lin])
    may, must, new, cbar, wq, wild = _frame_outcomes(warped["x_w"], warped["bar"], warped["sd"], warped["dsd"], F0, W0, depth, K, world2cam,
                                                     trunc, max_w, weight_scale)
    wild = wild | warped["ill"]
    all_skip = ~may.any(0)
    same = np.nanmax(np.where(may, new, -np.inf), 0) == np.nanmin(np.where(may, new, np.inf), 0)
    all_upd = must.all(0) & same & (wq.min(0) == wq.max(0))
    amb = wild | ~(all_skip | all_upd)
    # neighbour sets that are not forced: every admissible set's outcomes join the candidates
    w_lo = np.minimum(W0 + wq.min(0), max_w)
    w_hi = np.minimum(W0 + wq.max(0), max_w)
    extra = {}
    for i, alt in warped["alt"].items():
        amb[i] = True
        if alt is None:
            wild[i] = True
            continue
        p, b, sd, dsd, ill = alt
        k = len(sd)
        res = _frame_outcomes(p, b, sd, dsd, np.full(k, F0[i]), np.full(k, W0[i]), depth, K, world2cam, trunc, max_w, weight_scale)
        if ill.any() or res[5].any():
            wild[i] = True
            continue
        extra[i] = res
        w_lo[i] = min(w_lo[i], np.minimum(W0[i] + res[4].min(), max_w))
        w_hi[i] = max(w_hi[i], np.minimum(W0[i] + res[4].max(), max_w))
    upd = all_upd & ~amb
    return {"lin": lin, "upd": upd, "amb": amb, "new": new[0], "bar": cbar[0], "w_new": np.minimum(W0 + wq[0], max_w), "wild": wild,
            "may": may, "must": must, "cnew": new, "cbar": cbar, "wq": wq, "extra": extra, "w_lo": w_lo,
            "w_hi": w_hi, "max_w": int(max_w), "W0": W0}


def integrate_warped_check(prev, got, ref):
    """compares the volume words after the frame with integrate_warped64's prediction on its voxels.  Returns (violations, worst
    |got - new| / bar over updated unambiguous voxels, unambiguous updates, ambiguous voxels)"""
    lin = ref["lin"]
    prev = np.asarray(prev, np.uint32)[lin]
    got = np.asarray(got, np.uint32)[lin]
    Fg, Wg = halves(got)
    upd, amb = ref["upd"], ref["amb"]
    fixed = ~upd & ~amb
    bad = np.count_nonzero(got[fixed] != prev[fixed])
    bad += np.count_nonzero(Wg[upd] != ref["w_new"][upd])
    ratio = np.abs(Fg[upd] - ref["new"][upd]) / ref["bar"][upd]
    bad += np.count_nonzero(~(ratio <= 1.0))
    for i in np.flatnonzero(amb):
        if got[i] == prev[i] and not ref["must"][:, i].all():
            if i not in ref["extra"] or not ref["extra"][i][1].all():
                continue
        if ref["wild"][i]:
            if abs(Fg[i]) <= 1.0 and min(ref["W0"][i] + 1, ref["max_w"]) <= Wg[i] <= ref["max_w"]:
                continue
            if got[i] == prev[i]:
                continue
            bad += 1
            continue
        cands = [(ref["may"][:, i], ref["cnew"][:, i], ref["cbar"][:, i], ref["wq"][:, i])]
        if i in ref["extra"]:
            may, _, new, cbar, wq, _ = ref["extra"][i]
            cands.append((may.ravel(), new.ravel(), cbar.ravel(), wq.ravel()))
        hit = False
        for may, new, cbar, wq in cands:
            wn = np.minimum(ref["W0"][i] + wq, ref["max_w"])
            if np.any(may & (np.abs(Fg[i] - np.nan_to_num(new)) <= cbar) & (wn == Wg[i])):
                hit = True
                break
        bad += 0 if hit else 1
    return int(bad), float(ratio.max()) if len(ratio) else 0.0, int(upd.sum()), int(amb.sum())


# ------------------------------------------------------------------ search path --------------------------------------------------------------
def _half_diag(R, vs, ex, ey, ez):
    worst = 0.0
    for sy in (1, -1):
        for sz in (1, -1):
            e = R @ np.array([ex * vs[0], sy * ey * vs[1], sz * ez * vs[2]])
            worst = max(worst, np.linalg.norm(e))
    return 0.5 * worst * 1.001 + 1e-7


def search_path(nodes, dims, vs, vol2world, zchunk=None):
    """which search each block and run of df_integrate_warped takes.  A dict: block_n (node count of each block list), run_n (of each run
    list, -1 where the block has no list), run_block (each run's block), run_block_fits (its block list fits with room), and the fractions of runs that rank a list ('list'), walk the BVH ('tree') or the grid ('grid')"""
    Dx, Dy, Dz = (int(d) for d in dims)
    V = f64(nodes)[:, :3]
    M = len(V)
    vs = f64(vs)
    R, t = f64(vol2world[0]).reshape(3, 3), f64(vol2world[1]).reshape(3)
    zc = zchunk or (32 if Dz >= 64 else Dz)
    out = {"M": M, "block_n": [], "run_n": [], "run_block": [], "run_block_fits": []}
    if M > 8192:
        n_runs = -(-Dx // 8) * -(-Dy // 4) * -(-Dz // 8)
        out.update(list=0.0, tree=0.0, grid=1.0, runs=n_runs)
        return out
    if M < 8:
        out.update(list=0.0, tree=1.0, grid=0.0, runs=-(-Dx // 8) * -(-Dy // 4) * -(-Dz // 8))
        return out
    tree = cKDTree(V)
    hb = _half_diag(R, vs, 31.0, 7.0, zc - 1.0)
    h = _half_diag(R, vs, 7.0, 3.0, 7.0)
    n_list = n_tree = 0
    for bz in range(-(-Dz // zc)):
        z0, z1 = bz * zc, min(Dz, bz * zc + zc)
        for by in range(-(-Dy // 8)):
            for bx in range(-(-Dx // 32)):
                cb = R @ np.array([(bx * 32 + 15.5) * vs[0], (by * 8 + 3.5) * vs[1], (z0 + 0.5 * (zc - 1)) * vs[2]]) + t
                d8 = tree.query(cb, k=8)[0][-1]
                sel = tree.query_ball_point(cb, (d8 + 2 * hb) * 1.0002)
                nb = len(sel)
                out["block_n"].append(nb)
                fits = 8 <= nb <= 2048
                Vb = V[sel]
                sub = cKDTree(Vb) if fits else None
                for ya in range(by * 8, min(Dy, by * 8 + 8), 4):
                    for xa in range(bx * 32, min(Dx, bx * 32 + 32), 8):
                        for za in range(z0, z1, 8):
                            out["run_block"].append(len(out["block_n"]) - 1)
                            out["run_block_fits"].append(nb <= 0.5 * 2048 or M <= 0.5 * 2048)
                            if not fits:
                                n_tree += 1
                                out["run_n"].append(-1)
                                continue
                            c = R @ np.array([(xa + 3.5) * vs[0], (ya + 1.5) * vs[1], (za + 3.5) * vs[2]]) + t
                            r8 = sub.query(c, k=8)[0][-1]
                            nr = len(sub.query_ball_point(c, (r8 + 2 * h) * 1.0002))
                            out["run_n"].append(nr)
                            if nr <= 768:
                                n_list += 1
                            else:
                                n_tree += 1
    runs = n_list + n_tree
    out.update(list=n_list / runs, tree=n_tree / runs, grid=0.0, runs=runs)
    return out


def path_of(sp):
    """the case's search path where it holds by a wide margin.  The kernel's lists are at least as long as the restated ones (its radius is
    >= d8), so a list claimed to fit must fit with room: at most half its cap, or at most M when M itself is that small.  Overflows are
    claimed at 1.5 times the cap or more.
      list             90 % of the runs lie in a block whose list holds at most half of FUS_BLOCK_CAP (or M <= 0.5 FUS_BLOCK_CAP) and
                       hold at most half of FUS_LIST_CAP themselves;
      run_overflow     every block list fits (M <= 0.625 FUS_BLOCK_CAP: no list can be longer than M) and every run list holds 1.5
                       FUS_LIST_CAP or more (a run list is a subset of its block's, so the two margins cannot both be halves);
      block_overflow   every block list holds 1.5 FUS_BLOCK_CAP or more;
      tree (M < 8), grid (M > 8192); else mixed"""
    if sp["grid"] == 1.0:
        return "grid"
    if sp["M"] < 8:
        return "tree"
    bn = np.asarray(sp["block_n"])
    rn = np.asarray(sp["run_n"])
    if np.all(bn >= 1.5 * 2048):
        return "block_overflow"
    if sp["M"] <= 0.625 * 2048 and np.all(rn >= 1.5 * 768):
        return "run_overflow"
    block_fits = (bn <= 0.5 * 2048) | (sp["M"] <= 0.5 * 2048)
    runs_fit = np.asarray(sp["run_block_fits"]) & (rn >= 0) & (rn <= 0.5 * 768)
    if runs_fit.mean() >= 0.9 and np.all(block_fits[np.asarray(sp["run_block"])[runs_fit]]):
        return "list"
    return "mixed"


def straddle_runs(dims, vs, vol2cam, K, cols, rows, delta=1e-6, margin=16.0):
    """the runs (8 x 4 x 8 voxels) of df_integrate_warped whose visibility test only the camera-plane exit (`!(pc.z > 1e-2f)`) keeps from
    culling visible voxels: their box, grown by a voxel and by delta, has corners on both sides of the plane z = 1e-2 (not all behind
    z = -1e-3), and all eight corners project more than `margin` pixels beyond one image edge, while voxels of the run lie at least 2 cm in
    front of the camera and 2 pixels inside the image.  Float64 geometry with a margin, no field (identity or translation-only fields, for
    which the cull runs; delta is their displacement bound).  Returns [(run origin (x, y, z), voxels in view)]"""
    Dx, Dy, Dz = (int(d) for d in dims)
    vs = f64(vs)
    R, t = f64(vol2cam[0]).reshape(3, 3), f64(vol2cam[1]).reshape(3)
    fx, fy, cx, cy = f64(K)
    xw, yw, za = (a.ravel() for a in np.meshgrid(np.arange(0, Dx, 8), np.arange(0, Dy, 4), np.arange(0, Dz, 8), indexing="ij"))
    xb, yb, zb = np.minimum(xw + 7, Dx - 1), np.minimum(yw + 3, Dy - 1), np.minimum(za + 7, Dz - 1)
    pc = np.stack([np.stack([np.where(k & 1, (xb + 1) * vs[0] + delta, (xw - 1) * vs[0] - delta),
                             np.where(k & 2, (yb + 1) * vs[1] + delta, (yw - 1) * vs[1] - delta),
                             np.where(k & 4, (zb + 1) * vs[2] + delta, (za - 1) * vs[2] - delta)], 1) @ R.T + t for k in range(8)], 1)
    z = pc[..., 2]
    with np.errstate(divide="ignore", invalid="ignore"):
        u, v = fx * pc[..., 0] / z + cx, fy * pc[..., 1] / z + cy
    side = (u < -1 - margin).all(1) | (v < -1 - margin).all(1) | (u > cols + 1 + margin).all(1) | (v > rows + 1 + margin).all(1)
    out = []
    for r in np.flatnonzero(~(z < -1e-3).all(1) & (z <= 1e-2 - 1e-4).any(1) & side):
        gx, gy, gz = np.meshgrid(np.arange(xw[r], xb[r] + 1), np.arange(yw[r], yb[r] + 1), np.arange(za[r], zb[r] + 1), indexing="ij")
        P = np.stack([gx.ravel() * vs[0], gy.ravel() * vs[1], gz.ravel() * vs[2]], 1) @ R.T + t
        with np.errstate(divide="ignore", invalid="ignore"):
            uu, vv = fx * P[:, 0] / P[:, 2] + cx, fy * P[:, 1] / P[:, 2] + cy
        n = int(((P[:, 2] > 0.02) & (uu >= 2) & (uu < cols - 2) & (vv >= 2) & (vv < rows - 2)).sum())
        if n:
            out.append(((int(xw[r]), int(yw[r]), int(za[r])), n))
    return out

