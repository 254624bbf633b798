"""Float64 reference of the rigid TSDF stage: compute_dists_kernel (csrc/imgproc.cu), the integrate kernels, the ray-cast (csrc/tsdf.cu),
the cloud and normal extraction (csrc/extract.cu, csrc/volscan.cuh).  numpy only, no oracle call: it restates the operations, not the
float32 order of either implementation, so an operation both get wrong in the same way (an axis mix-up, a wrong offset) fails here.

Every float32 input (voxel size, truncation distance, intrinsics, poses) is taken at its float32 value and then computed on exactly in
float64.  U = 2^-24 is the unit roundoff of float32: one rounding of a value a errs by at most U |a|.

Distances (dists64).  The kernel forms finv = 1/f, xl = (x - cx) finv, a = xl^2 + yl^2, s = a + 1, its square root and d * lambda * 0.001f:
xl carries <= 3U (relative), its square 7U, a 8U, so s errs by 8U a + U s; the root halves that and adds U, the two products add 2.8U
(0.001f is 1e-3 within 0.8U): rel = 4U a / s + 4.5U in all.  A ray length whose interval r (1 +- rel) holds a rounding boundary of the half
is ambiguous: the half may be either neighbour.

Integration (integrate64).  A voxel (x, y, z) sits at P = (x vsx, y vsy, z vsz); its camera-space position is vc = R P + t, exactly.  The
kernels start from aff_mul(R, t, (x vsx, y vsy, 0)) (the products, three sums and the translation: <= 5U (sum_j |R_ij P_j| + |t_i|)) and add
zstep = R[:, 2] vsz z times.  Each addition rounds once, by at most U times the partial sum, and the partial sums are a linear walk between
the end points; zstep itself is off by U |zstep_i|.  So coordinate i drifts by at most
    eps_i = 5U (sum_j |R_ij P_j| + |t_i|) + z U (max(|vc_i(0)|, |vc_i(z)|) + |zstep_i|).
This is int5_domain_ok's bound (Dz + 8) 1.2e-7 B taken per voxel and per coordinate instead of at the volume's largest coordinate B.
Projection u = fx (X / Z) + cx moves by du = |fx| (eps_x + |X / Z| eps_z) / Z + U |fx X / Z| + U |u|, and v likewise.  The pixel index
(int)u and the image edges (u < 0, u >= cols) are one decision, floor(u), with integer thresholds: a voxel whose u lies within du of an
integer has two candidate columns, floor(u - du) and floor(u + du), and both are evaluated (four candidate pixels at most).  The sign
test Z > 0 is ambiguous within eps_z.  The signed distance sdf = Dp - |vc| moves by dsdf = sqrt(3) max_i eps_i + 3U |vc| + U |sdf| (the dot
product and the square root, then the difference); the gate sdf >= -trunc is ambiguous within dsdf.  A voxel is ambiguous only when its
candidates (pixel x gate outcome) lead to different results: a free-space voxel whose candidates all clamp to 1 is not.  Voxels whose
projection moves by a quarter pixel or more (next to the camera plane) are ambiguous with any outcome.
The update starts from the stored half h of the previous volume and its weight w: new = (h w + tsdf) / (w + 1), tsdf = min(1, sdf / trunc).
The kernel's tsdf errs by dsdf / trunc + 2U |tsdf| (the rounded 1 / trunc and the product), its fma and its division by U |new| each, so
before the final rounding to half the float32 value is within e = (dsdf / trunc + 2U) / (w + 1) + 2U |new| of new; the stored half is then
within bar = halfulp(|new| + e) + e of it, halfulp(a) being half the spacing of halves at a.  The weight of an unambiguous voxel is exact.

Ray-cast (raycast64).  The ray of pixel (x, y) is dir = normalize(R ((x - cx) / fx, (y - cy) / fy, 1)), org = t; the kernel's dir is within
24U of it per component (<= 3U on the reprojection, 3U sqrt(3) on the rotation, 6U on the normalisation).  The box clip restates
intersect() with the box [0, vs (D - 1)] and the reference's fmaxf(tmn.x, tmn.z) (equal to the maximum of the three, NaN-skipping as
fmaxf); an axis's t = (b - o) / d moves by |t| (3U + 24U / |d|), and tmin / tmax by the largest such move among the axes that can bind.
The march samples pos_k = org + dir (tmin + k step), fetched at rint(pos_k / vs) (round half to even), clamped.  The kernel's sample drifts
by eps_k,i = 24U t_k + |dir_i| dtmin + (k + 2) U max(|pos_0,i|, |pos_k,i|) + k U |vstep_i| (the chain of pos += vstep), in voxel units
eps / vs + 2U |q|.  A sample's candidate voxels (rint(q - dq), rint(q + dq) per axis) give the set of sign classes (< 0, = 0, > 0) it can
see; the ray is ambiguous where a pair test before it stops could take more than one outcome over those sets; so is tcurr_k = tmin + k step within k U (tcurr + step) + dtmin + dtmax of
tmax - step, and entering (tmin < tmax) within dtmin + dtmax.  On a hit the trilinear values Ft, Ftdt at the two samples move by
dF = sum_i L_i dq_i + 16U (L_i the largest edge difference along axis i of the cells q +- dq lie in; 16U the float32 sum of
eight products of four factors, |F| <= 1), and
Ts = tcurr - step Ft / (Ftdt - Ft) by dTs = dtcurr + step (dFt / |D| + |Ft| (dFt + dFtdt) / D^2) + 4U (|Ts| + step |Ft / D|), D = Ftdt - Ft;
the vertex org + dir Ts by 24U |Ts| + |dir_i| dTs + U (|dir_i Ts| + |v_i|).  The normal's six samples at vertex +- gd e_i move together
with the vertex, so that common shift cancels in g_i = (F+ - F-) / gd_i up to how much g itself changes: it is taken as the largest change of
g over the eight corners vertex +- dv (g is multilinear between grid planes and the box is about a thousandth of a voxel); each sample's
own rounding adds its dF, and n = g / |g| moves by 2 |dg| / |g| + 4U.  The outputs Rinv (v - org) and
Rinv n add their propagated error through |Rinv| and 3U of rounding.  The bound on Ts is first order: a ray whose (dFt + dFtdt) / |D|
exceeds 0.1 is ambiguous; so is one whose |dg| / |g| exceeds 0.5 (|n(g) - n(h)| <= 2 |g - h| / |g| holds at any size, but a bar near 1
checks nothing), and one whose interpolation stencils lie within dq of the box [0, D - 1) that decides NaN.

Extraction (extract64, normals64).  The crossing rule reads stored halves only, so the points, their count and their (z, y, x, axis) order
are exact.  A point's volume coordinates are positive sums and products of (x + 1/2) vs, |F| and |Fn| (<= 8U relative) and the pose adds
3U of its own: each coordinate is within 16U (sum_j |R_ij p_j| + |t_i|).  The normals take the extracted float32 points as input:
point = Rinv (p - t) errs by U |p - t| + 3U sum_j |Rinv_ij (p - t)_j|, the index test gx > 1 .. gx < Dx - 2 is ambiguous where rint's two
candidates straddle it, and the rotated gradient R g is normalised as the ray-cast's normal is.
"""
from __future__ import annotations

import numpy as np

U = 2.0 ** -24
AMB_FIRST_ORDER = 0.1                   # (dFt + dFtdt) / |Ftdt - Ft| above this: the first-order bound on Ts is not trusted, the ray is ambiguous
AMB_GRADIENT = 0.5                      # |dg| / |g| above this: the normal's bar (2 |dg| / |g|) says nothing, the ray or point is ambiguous


def f64(a):
    """float32 values (the kernels' parameters) in float64"""
    return np.asarray(a, np.float32).astype(np.float64)


def halves(vol):
    """(F as float64, W) of volume words"""
    vol = np.asarray(vol, np.uint32)
    return (vol & 0xffff).astype(np.uint16).view(np.float16).astype(np.float64), (vol >> 16).astype(np.int64)


def halfulp(a):
    """half the spacing of float16 values at |a| (subnormal spacing below 2^-14)"""
    _, e = np.frexp(np.maximum(np.abs(a), 2.0 ** -14))
    return np.ldexp(1.0, e - 12)


# ------------------------------------------------------------------ distances -------------------------------------------------------------
def dists64(depth, K):
    """(ray length in metres, the half bits it rounds to, ambiguous) of a u16 millimetre depth image"""
    fx, fy, cx, cy = f64(K)
    rows, cols = depth.shape
    xl = (np.arange(cols) - cx) / fx
    yl = (np.arange(rows) - cy) / fy
    a = xl[None, :] ** 2 + yl[:, None] ** 2
    r = depth.astype(np.float64) * np.sqrt(a + 1.0) * 1e-3
    h = r.astype(np.float16)
    rel = 4 * U * a / (a + 1) + 4.5 * U
    amb = (r * (1 - rel)).astype(np.float16) != (r * (1 + rel)).astype(np.float16)
    return r, h.view(np.uint16), amb


# ------------------------------------------------------------------ integration -----------------------------------------------------------
def _voxel_positions(dims, vs, R, t, zs=None):
    Dx, Dy, Dz = (int(d) for d in dims)
    z, y, x = np.meshgrid(np.arange(Dz) if zs is None else zs, np.arange(Dy), np.arange(Dx), indexing="ij")
    P = np.stack([x.ravel() * vs[0], y.ravel() * vs[1], z.ravel() * vs[2]])
    return P, z.ravel()


def integrate64(prev, dims, vs, trunc, max_w, dists, vol2cam, K):
    """one frame's update of the volume words `prev` (flat, (z, y, x) order) by the u16 half image `dists`.  Returns a dict:
    upd (unambiguous voxels that are updated), amb (ambiguous voxels), new (predicted F of updated voxels), bar (their bar), w_new, and the
    candidates of the ambiguous voxels (cand_ok [4, n], cand_new [4, n], cand_bar [4, n], may_skip [n], wild [n])"""
    vs, R, t = f64(vs), f64(vol2cam[0]).reshape(3, 3), f64(vol2cam[1]).reshape(3)
    fx, fy, cx, cy = f64(K)
    trunc = float(np.float32(trunc))
    rows, cols = dists.shape
    D = np.asarray(dists, np.uint16).view(np.float16).astype(np.float64)
    F0, W0 = halves(prev)
    P, z = _voxel_positions(dims, vs, R, t)
    vc = R @ P + t[:, None]
    P0 = P.copy(); P0[2] = 0
    vc0 = R @ P0 + t[:, None]
    zstep = R[:, 2] * vs[2]
    eps = 5 * U * (np.abs(R) @ np.abs(P0) + np.abs(t)[:, None]) + z * U * (np.maximum(np.abs(vc0), np.abs(vc)) + np.abs(zstep)[:, None])
    X, Y, Z = vc
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        qx, qy = X / Z, Y / Z
        u, v = fx * qx + cx, fy * qy + cy
        du = abs(fx) * (eps[0] + np.abs(qx) * eps[2]) / np.abs(Z) + U * np.abs(fx * qx) + U * np.abs(u)
        dv = abs(fy) * (eps[1] + np.abs(qy) * eps[2]) / np.abs(Z) + U * np.abs(fy * qy) + U * np.abs(v)
    front = Z > eps[2]                                   # certainly in front of the camera plane
    maybe = Z > -eps[2]
    with np.errstate(invalid="ignore"):
        off = (u + du < 0) | (u - du >= cols) | (v + dv < 0) | (v - dv >= rows)     # off the image for every candidate
    wild = maybe & ~off & ~((du < 0.25) & (dv < 0.25))  # projection too unstable to name candidates: any outcome
    norm = np.sqrt((vc * vc).sum(0))
    dsdf_pos = np.sqrt(3.0) * eps.max(0) + 3 * U * norm
    sane = maybe & ~wild & ~off
    ul, uh = np.full(z.shape, -1, np.int64), np.full(z.shape, -1, np.int64)
    vl, vh = ul.copy(), uh.copy()
    ul[sane], uh[sane] = np.floor(u[sane] - du[sane]), np.floor(u[sane] + du[sane])
    vl[sane], vh[sane] = np.floor(v[sane] - dv[sane]), np.floor(v[sane] + dv[sane])
    inv_t = 1.0 / trunc
    cand_must, cand_may, cand_new, cand_bar = [], [], [], []
    for cu, cv in ((ul, vl), (uh, vl), (ul, vh), (uh, vh)):
        ok = sane & (cu >= 0) & (cu < cols) & (cv >= 0) & (cv < rows)
        Dp = np.zeros(z.shape)
        Dp[ok] = D[cv[ok], cu[ok]]
        live = ok & (Dp != 0)
        sdf = Dp - norm
        dsdf = dsdf_pos + U * np.abs(sdf)
        must = live & front & (sdf > -trunc + dsdf)
        may = live & maybe & (sdf >= -trunc - dsdf)
        tsdf = np.minimum(1.0, sdf * inv_t)
        new = (F0 * W0 + tsdf) / (W0 + 1)
        e = (dsdf * inv_t + 2 * U) / (W0 + 1) + 2 * U * np.abs(new)
        cand_must.append(must); cand_may.append(may); cand_new.append(np.where(may, new, np.nan)); cand_bar.append(halfulp(np.abs(new) + e) + e)
    cand_must, cand_may, cand_new, cand_bar = (np.stack(a) for a in (cand_must, cand_may, cand_new, cand_bar))
    # one outcome for every candidate: all skip for certain, or all update for certain with the same tsdf (free space clamps to 1)
    all_skip = ~cand_may.any(0)
    all_upd = cand_must.all(0) & (np.nanmax(np.where(cand_may, cand_new, -np.inf), 0) == np.nanmin(np.where(cand_may, cand_new, np.inf), 0))
    amb = wild | ~(all_skip | all_upd)
    upd = all_upd & ~amb
    return {"upd": upd, "amb": amb, "new": cand_new[0], "bar": cand_bar[0], "w_new": np.minimum(W0 + 1, int(max_w)),
            "cand_ok": cand_may, "cand_new": cand_new, "cand_bar": cand_bar, "may_skip": ~cand_must.all(0), "wild": wild, "max_w": int(max_w)}


def integrate_check(prev, got, ref):
    """compares the volume words after the frame with integrate64's prediction `ref`.  Returns (violations, worst |got - new| / bar over
    updated unambiguous voxels, unambiguous updates, ambiguous voxels)"""
    prev = np.asarray(prev, np.uint32)
    got = np.asarray(got, np.uint32)
    Fg, Wg = halves(got)
    upd, amb = ref["upd"], ref["amb"]
    fixed = ~upd & ~amb
    bad = np.count_nonzero(got[fixed] != prev[fixed])                      # certainly skipped: untouched, bit for bit
    bad += np.count_nonzero(Wg[upd] != ref["w_new"][upd])
    ratio = np.abs(Fg[upd] - ref["new"][upd]) / ref["bar"][upd]
    bad += np.count_nonzero(~(ratio <= 1.0))
    ia = np.flatnonzero(amb)
    if len(ia):
        same = got[ia] == prev[ia]
        skip_ok = same & ref["may_skip"][ia]
        w_ok = Wg[ia] == ref["w_new"][ia]
        near = np.abs(Fg[ia][None, :] - ref["cand_new"][:, ia]) <= ref["cand_bar"][:, ia]
        upd_ok = w_ok & ((ref["cand_ok"][:, ia] & near).any(0) | (ref["wild"][ia] & (np.abs(Fg[ia]) <= 1.0)))
        bad += np.count_nonzero(~(skip_ok | upd_ok))
    return int(bad), float(ratio.max()) if len(ratio) else 0.0, int(upd.sum()), int(amb.sum())


# ------------------------------------------------------------------ which integrate kernel -------------------------------------------------
def _int5_domain_ok(dims, vs, trunc, vol2cam, K, cols, rows, pitch):
    """int5_domain_ok (csrc/tsdf.cu), restated: the float comparisons in float32, B and the drift bound in double"""
    f = np.float32
    a = [f(v) for v in np.concatenate([np.asarray(vol2cam[0], np.float32).reshape(9), np.asarray(vol2cam[1], np.float32).reshape(3)])]
    if not all(abs(v) < f(1e6) for v in a):
        return False
    rmax, tmax = max(abs(v) for v in a[:9]), max(abs(v) for v in a[9:])
    vs = [f(v) for v in vs]
    if not all(f(1e-9) < v < f(1e3) for v in vs):
        return False
    Dx, Dy, Dz = (int(d) for d in dims)
    B = float(tmax) + 3.0 * float(rmax) * (Dx * float(vs[0]) + Dy * float(vs[1]) + Dz * float(vs[2])) * 1.001
    if not B < 64.0 or not (Dz + 8) * 1.2e-7 * B < 4e-3:
        return False
    fx, fy, cx, cy = (f(k) for k in K)
    if not (abs(fx) < f(1e6) and abs(fy) < f(1e6)):
        return False
    if not (f(1) <= abs(cx) < f(1e6) and f(1) <= abs(cy) < f(1e6)):
        return False
    tr = f(trunc)
    tinv = f(1) / tr
    if not (f(1e-9) < tr < f(1e3) and f(0) < tinv < f(1e12)):
        return False
    if not (0 < cols <= 32768 and 0 < rows <= 32768) or pitch * rows >= 0x7fffffff or Dx * Dy * Dz >= 0x7fffffff:
        return False
    return True


def integrate_kernel_for(dims, impl, K, vol2cam, vs, trunc, cols, rows, pitch, aligned=True):
    """(kernel, vx, zchunk) df_integrate_tracked launches: kernel 5 (packed), 3 (scalar with culling) or 0 (plain integrate_kernel<vx>)"""
    Dx, Dy, Dz = (int(d) for d in dims)
    zchunk = 64 if Dz >= 256 else (32 if Dz >= 64 else Dz)
    vec4 = Dx % 4 == 0 and aligned
    if impl in (3, 5) and vec4 and Dx % 32 == 0 and Dy % 16 == 0:
        return (5 if impl == 5 and _int5_domain_ok(dims, vs, trunc, vol2cam, K, cols, rows, pitch) else 3), 4, zchunk
    return 0, (4 if vec4 else 1), zchunk


# ------------------------------------------------------------------ ray-cast --------------------------------------------------------------
def _interp(F, dims, q, dq=None):
    """trilinear interpolation of the (z, y, x) float64 volume F at voxel coordinates q [3, n]; NaN outside [0, D - 1).  With dq, also a
    bound on how far it moves when q moves by dq: per axis the largest edge difference of the cells q - dq and q + dq fall in (trilinear
    interpolation is multilinear in a cell), plus 16U for the float32 sum of eight products of four factors (|F| <= 1)."""
    Dx, Dy, Dz = (int(d) for d in dims)
    hi = np.array([Dx - 2, Dy - 2, Dz - 2])[:, None]
    g = np.floor(q)
    ok = (g[0] >= 0) & (g[1] >= 0) & (g[2] >= 0) & (g[0] < Dx - 1) & (g[1] < Dy - 1) & (g[2] < Dz - 1)
    out = np.full(q.shape[1], np.nan)
    if ok.any():
        gx, gy, gz = (g[i][ok].astype(np.int64) for i in range(3))
        a, b, c = (q[i][ok] - g[i][ok] for i in range(3))
        s = 0.0
        for dz, wz in ((0, 1 - c), (1, c)):
            for dy, wy in ((0, 1 - b), (1, b)):
                for dx, wx in ((0, 1 - a), (1, a)):
                    s = s + F[gz + dz, gy + dy, gx + dx] * wx * wy * wz
        out[ok] = s
    if dq is None:
        return out
    slope = np.zeros_like(q)
    for cell in (np.clip(np.floor(q - dq), 0, hi), np.clip(np.floor(q + dq), 0, hi)):
        cx, cy, cz = (np.nan_to_num(cell[i]).astype(np.int64) for i in range(3))
        for o in range(4):
            e1, e2 = o & 1, o >> 1
            slope[0] = np.fmax(slope[0], np.abs(F[cz + e2, cy + e1, cx + 1] - F[cz + e2, cy + e1, cx]))
            slope[1] = np.fmax(slope[1], np.abs(F[cz + e2, cy + 1, cx + e1] - F[cz + e2, cy, cx + e1]))
            slope[2] = np.fmax(slope[2], np.abs(F[cz + 1, cy + e2, cx + e1] - F[cz, cy + e2, cx + e1]))
    return out, (slope * dq).sum(0) + 16 * U


def _near_box(q, dq, dims):
    """a coordinate within dq of 0 or D - 1, where the interpolation's NaN decision flips"""
    D = np.asarray(dims, np.float64)[:, None] - 1
    return ((np.abs(q) <= dq) | (np.abs(q - D) <= dq)).any(0)


def _sign_class(F, dims, q, dq):
    """the sign classes (bit 0: < 0, bit 1: = 0, bit 2: > 0) the fetch of q can see: its candidate voxels rint(q +- dq), clamped"""
    Dx, Dy, Dz = (int(d) for d in dims)
    hi = np.array([Dx - 1, Dy - 1, Dz - 1])[:, None]
    lo_i = np.clip(np.rint(q - dq), 0, hi).astype(np.int64)
    hi_i = np.clip(np.rint(q + dq), 0, hi).astype(np.int64)
    nom = np.clip(np.rint(q), 0, hi).astype(np.int64)
    cls = 1 << (np.sign(F[nom[2], nom[1], nom[0]]).astype(np.int64) + 1)
    split = np.flatnonzero((lo_i != hi_i).any(0))
    for k in range(8):
        sel = [(hi_i if (k >> i) & 1 else lo_i)[i][split] for i in range(3)]
        cls[split] |= 1 << (np.sign(F[sel[2], sel[1], sel[0]]).astype(np.int64) + 1)
    return cls


def _pair(a, b):
    """(hit, stop, undecided) of the march's pair test on class sets a, b: hit = (> 0, < 0), stop = (< 0, > 0), undecided when more than
    one outcome is possible"""
    hit_may, stop_may = ((a & 4) != 0) & ((b & 1) != 0), ((a & 1) != 0) & ((b & 4) != 0)
    hit_must, stop_must = (a == 4) & (b == 1), (a == 1) & (b == 4)
    none_may = ~(hit_must | stop_must)
    n = hit_may.astype(int) + stop_may + none_may
    return hit_must, stop_must, n > 1


def _gradient(F, dims, vs, gd, V, dV):
    """(g, dg, near box) of the central differences at the volume positions V [3, n] whose float32 counterparts lie within dV of them.
    The six samples move together with the vertex, so their common shift is taken from g itself at the eight corners V +- dV (g is
    multilinear between grid planes, and the box is a thousandth of a voxel); each sample's own rounding adds U |p| / vs + 2U |q|."""
    def central(P):
        g = np.zeros_like(P)
        near = np.zeros(P.shape[1], bool)
        for a in range(3):
            Fs = []
            for sgn in (1.0, -1.0):
                p = P.copy()
                p[a] += sgn * gd[a]
                qs = p / vs[:, None]
                near |= _near_box(qs, dV / vs[:, None] + 3 * U * np.abs(qs), dims)
                Fs.append(_interp(F, dims, qs))
            g[a] = (Fs[0] - Fs[1]) / gd[a]
        return g, near
    g, near = central(V)
    shift = np.zeros_like(g)
    for k in range(8):
        s = np.array([1.0 if (k >> i) & 1 else -1.0 for i in range(3)])[:, None]
        gk, _ = central(V + s * dV)
        shift = np.fmax(shift, np.abs(gk - g))
    own = 2 * (2 * ((U * np.abs(V) + gd[:, None] * U) / vs[:, None] + 2 * U * np.abs(V / vs[:, None])).sum(0) + 16 * U)
    return g, shift + own / gd[:, None] + 3 * U * np.abs(g), near


def raycast64(vol, dims, vs, trunc, cam2vol, Rinv, K, cols, rows, step_factor, delta_factor, pixels=None):
    """the ray-cast of the pixels (flat indices y * cols + x; all when None).  Returns a dict: pix, hit, amb, vertex [n, 3], normal [n, 3]
    (NaN where no hit), vbar, nbar (per component)"""
    Dx, Dy, Dz = (int(d) for d in dims)
    F, _ = halves(vol)
    F = F.reshape(Dz, Dy, Dx)
    vs, R, org = f64(vs), f64(cam2vol[0]).reshape(3, 3), f64(cam2vol[1]).reshape(3)
    Ri = f64(Rinv).reshape(3, 3)
    fx, fy, cx, cy = f64(K)
    step = float(np.float32(trunc)) * float(np.float32(step_factor))
    gd = vs * float(np.float32(delta_factor))
    pix = np.arange(cols * rows) if pixels is None else np.asarray(pixels, np.int64)
    n = len(pix)
    x, y = (pix % cols).astype(np.float64), (pix // cols).astype(np.float64)
    rp = np.stack([(x - cx) / fx, (y - cy) / fy, np.ones(n)])
    d = R @ rp
    d /= np.sqrt((d * d).sum(0))
    ddir = 24 * U
    box = vs * (np.array([Dx, Dy, Dz]) - 1)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        inv = 1.0 / d
        tbot = inv * (0.0 - org[:, None])
        ttop = inv * (box[:, None] - org[:, None])
        tmn, tmx = np.fmin(ttop, tbot), np.fmax(ttop, tbot)
        tmin = np.fmax(np.fmax(tmn[0], tmn[1]), np.fmax(tmn[0], tmn[2]))
        tmax = np.fmin(np.fmin(tmx[0], tmx[1]), np.fmin(tmx[0], tmx[2]))
        dt_mn = np.abs(tmn) * (3 * U + ddir / np.abs(d))
        dt_mx = np.abs(tmx) * (3 * U + ddir / np.abs(d))
        dtmin = np.nanmax(np.where(tmn + dt_mn >= tmin, dt_mn, 0.0), 0)
        dtmax = np.nanmax(np.where(tmx - dt_mx <= tmax, dt_mx, 0.0), 0)
    dtmin = np.where(tmin > 0, dtmin, 0.0)
    tmin = np.fmax(0.0, tmin)
    enter = tmin < tmax
    amb = (enter != (tmin < tmax + dtmin + dtmax)) | (enter != (tmin < tmax - dtmin - dtmax))
    tend = tmax - step
    dtend = dtmax + U * (abs(tmax) + step)
    hit = np.zeros(n, bool)
    khit = np.zeros(n, np.int64)

    def sample(i, k):
        tk = tmin[i] + k * step
        p = org[:, None] + d[:, i] * tk
        p0 = org[:, None] + d[:, i] * tmin[i]
        e = (ddir * tk + np.abs(d[:, i]) * dtmin[i] + (k + 2) * U * np.maximum(np.abs(p0), np.abs(p))
             + k * U * np.abs(d[:, i] * step) + U * np.abs(d[:, i] * tmin[i]))
        q = p / vs[:, None]
        return q, e / vs[:, None] + 2 * U * np.abs(q)

    act = np.flatnonzero(enter & ~amb)
    q, dq = sample(act, 0)
    c_curr = _sign_class(F, dims, q, dq)
    k = 0
    while len(act):
        tc = tmin[act] + k * step
        dtc = dtmin[act] + k * U * (np.abs(tc) + step)
        go = tc < tend[act]
        undecided = (go != (tc < tend[act] + dtc + dtend[act])) | (go != (tc < tend[act] - dtc - dtend[act]))
        q, dq = sample(act, k + 1)
        c_next = _sign_class(F, dims, q, dq)
        found, stop, split = _pair(c_curr, c_next)
        undecided |= go & split
        found &= go
        hit[act[found]] = True
        khit[act[found]] = k
        done = ~go | stop | found | undecided
        amb[act[undecided]] = True
        keep = ~done
        act, c_curr = act[keep], c_next[keep]
        k += 1
    vertex = np.full((n, 3), np.nan)
    normal = np.full((n, 3), np.nan)
    vbar = np.full((n, 3), np.nan)
    nbar = np.full((n, 3), np.nan)
    ih = np.flatnonzero(hit & ~amb)
    if len(ih):
        kk = khit[ih]
        qc, dqc = sample(ih, kk)
        qn, dqn = sample(ih, kk + 1)
        (Ft, dFt), (Ftdt, dFtdt) = _interp(F, dims, qc, dqc), _interp(F, dims, qn, dqn)
        Dd = Ftdt - Ft
        tc = tmin[ih] + kk * step
        dtc = dtmin[ih] + kk * U * (np.abs(tc) + step)
        with np.errstate(divide="ignore", invalid="ignore"):
            r = Ft / Dd
            Ts = tc - step * r
            dTs = dtc + step * (dFt / np.abs(Dd) + np.abs(Ft) * (dFt + dFtdt) / Dd ** 2) + 4 * U * (np.abs(Ts) + step * np.abs(r))
            bad = ~((dFt + dFtdt) / np.abs(Dd) <= AMB_FIRST_ORDER) & np.isfinite(Ft) & np.isfinite(Ftdt)
        bad |= _near_box(qc, dqc, dims) | _near_box(qn, dqn, dims)
        dv = d[:, ih]
        V = org[:, None] + dv * Ts
        dV = ddir * np.abs(Ts) + np.abs(dv) * dTs + U * (np.abs(dv * Ts) + np.abs(V))
        g, dg, near = _gradient(F, dims, vs, gd, V, dV)
        bad |= near
        gn = np.sqrt((g * g).sum(0))
        with np.errstate(divide="ignore", invalid="ignore"):
            rel = np.sqrt((dg * dg).sum(0)) / gn
            bad |= ~(rel <= AMB_GRADIENT) & np.isfinite(gn)
            nn = g / gn
        dn = 2 * rel + 4 * U
        ok = np.isfinite(nn).all(0)
        amb[ih[bad]] = True
        keep = ~bad
        hit[ih[~ok & keep]] = False
        sel = ok & keep
        hs = ih[sel]
        Vo = V[:, sel] - org[:, None]
        vertex[hs] = (Ri @ Vo).T
        vbar[hs] = (np.abs(Ri) @ (dV[:, sel] + U * np.abs(Vo)) + 3 * U * (np.abs(Ri) @ np.abs(Vo))).T
        normal[hs] = (Ri @ nn[:, sel]).T
        nbar[hs] = (np.abs(Ri) @ np.broadcast_to(dn[sel], (3, len(hs))) + 3 * U * (np.abs(Ri) @ np.abs(nn[:, sel]))).T
    hit &= ~amb
    return {"pix": pix, "hit": hit, "amb": amb, "vertex": vertex, "normal": normal, "vbar": vbar, "nbar": nbar}


def raycast_check(points, normals, ref):
    """compares the kernel's maps (rows, cols, 4) on ref's pixels.  Returns (hit/miss disagreements, worst vertex ratio, worst normal ratio,
    unambiguous hits, ambiguous rays)"""
    P = np.asarray(points, np.float64).reshape(-1, 4)[ref["pix"], :3]
    N = np.asarray(normals, np.float64).reshape(-1, 4)[ref["pix"], :3]
    ghit = ~np.isnan(P[:, 0])
    una = ~ref["amb"]
    bad = int(np.count_nonzero(ghit[una] != ref["hit"][una]))
    h = una & ref["hit"] & ghit
    rv = np.abs(P[h] - ref["vertex"][h]) / ref["vbar"][h]
    rn = np.abs(N[h] - ref["normal"][h]) / ref["nbar"][h]
    rv_max = float(rv.max()) if rv.size else 0.0
    rn_max = float(rn.max()) if rn.size else 0.0
    bad += int(np.count_nonzero(~(rv <= 1.0)) + np.count_nonzero(~(rn <= 1.0)))
    return bad, rv_max, rn_max, int(h.sum()), int(ref["amb"].sum())


# ------------------------------------------------------------------ extraction ------------------------------------------------------------
def extract64(vol, dims, vs, pose):
    """the cloud points in the extraction's (z, y, x, axis) order: (points [n, 3], bars [n, 3], voxel index [n], axis [n])"""
    Dx, Dy, Dz = (int(d) for d in dims)
    vs, R, t = f64(vs), f64(pose[0]).reshape(3, 3), f64(pose[1]).reshape(3)
    F, W = halves(vol)
    F, W = F.reshape(Dz, Dy, Dx), W.reshape(Dz, Dy, Dx)
    act = (W != 0) & (F != 1.0)
    keys, pts = [], []
    zz, yy, xx = np.meshgrid(np.arange(Dz), np.arange(Dy), np.arange(Dx), indexing="ij")
    for a in range(3):
        sl = [slice(0, Dz - 1), slice(None), slice(None)]
        nb = [slice(1, Dz), slice(None), slice(None)]
        if a == 0:
            sl[2], nb[2] = slice(0, Dx - 1), slice(1, Dx)
            nb[0] = slice(0, Dz - 1)
        elif a == 1:
            sl[1], nb[1] = slice(0, Dy - 1), slice(1, Dy)
            nb[0] = slice(0, Dz - 1)
        sl, nb = tuple(sl), tuple(nb)
        f, fn = F[sl], F[nb]
        m = act[sl] & act[nb] & (((f > 0) & (fn < 0)) | ((f < 0) & (fn > 0)))
        x, y, z = xx[sl][m], yy[sl][m], zz[sl][m]
        af, afn = np.abs(f[m]), np.abs(fn[m])
        V = np.stack([(x + 0.5) * vs[0], (y + 0.5) * vs[1], (z + 0.5) * vs[2]])
        V[a] = (V[a] * afn + (V[a] + vs[a]) * af) / (af + afn)
        keys.append((z * Dy + y) * Dx + x)
        pts.append((V, np.full(len(x), a)))
    lin = np.concatenate(keys)
    axis = np.concatenate([p[1] for p in pts])
    V = np.concatenate([p[0] for p in pts], axis=1)
    order = np.lexsort((axis, lin))
    V, lin, axis = V[:, order], lin[order], axis[order]
    out = (R @ V + t[:, None]).T
    bar = (16 * U * (np.abs(R) @ np.abs(V) + np.abs(t)[:, None])).T
    return out, bar, lin, axis


def normals64(vol, dims, vs, pts, pose, Rinv, delta_factor):
    """the normals of the float32 cloud points pts [n, >= 3].  Returns (normals [n, 3] (NaN outside the index test), bars [n, 3], ambiguous)"""
    Dx, Dy, Dz = (int(d) for d in dims)
    F, _ = halves(vol)
    F = F.reshape(Dz, Dy, Dx)
    vs, R, t = f64(vs), f64(pose[0]).reshape(3, 3), f64(pose[1]).reshape(3)
    Ri = f64(Rinv).reshape(3, 3)
    gd = vs * float(np.float32(delta_factor))
    p = np.asarray(pts, np.float64)[:, :3].T
    dpt = p - t[:, None]
    point = Ri @ dpt
    dpoint = U * (np.abs(Ri) @ np.abs(dpt)) + 3 * U * (np.abs(Ri) @ np.abs(dpt))
    q = point / vs[:, None]
    dq = dpoint / vs[:, None] + 2 * U * np.abs(q)
    lim = np.array([Dx, Dy, Dz])[:, None] - 2

    def inside(g):
        return ((g > 1) & (g < lim)).all(0)
    ins = inside(np.rint(q))
    amb = inside(np.rint(q - dq)) != inside(np.rint(q + dq))
    n = p.shape[1]
    g = np.full((3, n), np.nan)
    dg = np.zeros((3, n))
    for a in range(3):
        Fs, dFs = [], []
        for sgn in (1.0, -1.0):
            s = point.copy()
            s[a] += sgn * gd[a]
            qs = s / vs[:, None]
            dqs = (dpoint + U * np.abs(s)) / vs[:, None] + 2 * U * np.abs(qs)
            Fv, dFv = _interp(F, dims, qs, dqs)
            Fs.append(Fv)
            dFs.append(dFv)
        g[a] = (Fs[0] - Fs[1]) / gd[a]
        dg[a] = (dFs[0] + dFs[1]) / gd[a] + 3 * U * np.abs(g[a])
    Rg = R @ g
    dRg = np.abs(R) @ dg + 3 * U * (np.abs(R) @ np.abs(g))
    gn = np.sqrt((Rg * Rg).sum(0))
    with np.errstate(divide="ignore", invalid="ignore"):
        rel = np.sqrt((dRg * dRg).sum(0)) / gn
        nrm = Rg / gn
    amb |= ins & ~(rel <= AMB_GRADIENT)
    nrm[:, ~ins] = np.nan
    bar = np.broadcast_to(2 * rel + 4 * U, (3, n)).T.copy()
    return nrm.T, bar, amb
