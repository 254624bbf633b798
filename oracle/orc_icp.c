/* CPU ORACLE (test infrastructure only) -- projective point-to-plane ICP.
 * Restates kfusion/src/cuda/proj_icp.cu (points variant, USE_DEPTH off) and
 * kfusion/src/projective_icp.cpp of the reference.  PARITY UNPINNED by the reference (no ICP tests, and
 * cv::solve/cv::determinant/Affine3f(rvec,t) live in OpenCV 2.4.13, absent here): the 6x6 solve below is a
 * double-precision symmetric-eigen pseudo-inverse (what DECOMP_SVD computes for a symmetric matrix). */
#include "orc_common.h"
#include <float.h>

/* ComputeIcpHelper::find_coresp (points variant), proj_icp.cu:80-108; row build :359-368.  The rule for one pixel (x, y):
 * returns the linear index v * cols + u of the matched previous pixel and writes the 7-float row, or returns -1 when the pixel
 * is rejected (row untouched). */
static long long icp_row_points(const float *vcurr, size_t vcpitch, const float *ncurr, size_t ncpitch, const float *vprev, size_t vppitch,
                                const float *nprev, size_t nppitch, int cols, int rows, orc_intr k, const orc_aff3f *T,
                                float dist2_thres, float min_cosine, int x, int y, float row[7])
{
    const float *vc = orc_row_f4(vcurr, vcpitch, y) + 4 * x;
    orc_f3 s = f3(vc[0], vc[1], vc[2]);
    if (isnan(s.x)) return -1;
    s = orc_aff_mul(T, s);
    float u = fmaf(k.fx, s.x / s.z, k.cx);
    float v = fmaf(k.fy, s.y / s.z, k.cy);
    if (s.z <= 0 || u < 0 || v < 0 || u >= (float)cols || v >= (float)rows) return -1;
    if (!(u == u) || !(v == v)) return -1;
    const float *dp = orc_row_f4(vprev, vppitch, (int)v) + 4 * (int)u;
    orc_f3 d = f3(dp[0], dp[1], dp[2]);
    if (isnan(d.x)) return -1;
    orc_f3 df = orc_sub(s, d);
    float dist2 = orc_dot(df, df);
    if (dist2 > dist2_thres) return -1;
    const float *nc = orc_row_f4(ncurr, ncpitch, y) + 4 * x;
    orc_f3 ns = orc_mat_mul(T->R, f3(nc[0], nc[1], nc[2]));
    const float *np = orc_row_f4(nprev, nppitch, (int)v) + 4 * (int)u;
    orc_f3 nd = f3(np[0], np[1], np[2]);
    float cosine = fabsf(orc_dot(ns, nd));
    if (!(cosine >= min_cosine)) { if (cosine < min_cosine) return -1; }   /* NaN cosine passes, as in the reference */
    orc_f3 c = orc_cross(s, nd);
    row[0] = c.x; row[1] = c.y; row[2] = c.z; row[3] = nd.x; row[4] = nd.y; row[5] = nd.z;
    row[6] = orc_dot(nd, orc_sub(d, s));
    return (long long)(int)v * cols + (int)u;
}

/* ComputeIcpHelper::find_coresp, USE_DEPTH variant (proj_icp.cu:47-78; compiled in when internal.hpp:6 defines USE_DEPTH):
 * the source point is the current depth pixel (u16 millimetres) re-projected with finv = 1/f (reproj, proj_icp.cu:39-45), the
 * destination is the previous depth map point-sampled at the projection (texture<ushort> dprev_tex, cudaFilterModePoint) and
 * re-projected at the fractional coordinates; normals as in the points variant.  Same return value and row as icp_row_points. */
static long long icp_row_depth(const unsigned short *dcurr, size_t dcpitch, const float *ncurr, size_t ncpitch, const unsigned short *dprev,
                               size_t dppitch, const float *nprev, size_t nppitch, int cols, int rows, orc_intr k, const orc_aff3f *T,
                               float dist2_thres, float min_cosine, int x, int y, float row[7])
{
    const float finvx = 1.f / k.fx, finvy = 1.f / k.fy;              /* setLevelIntr, projective_icp.cpp:22 */
    const int src_z = ((const unsigned short *)((const char *)dcurr + (size_t)y * dcpitch))[x];
    if (src_z == 0) return -1;
    const float zs = src_z * 0.001f;
    orc_f3 s = f3(zs * ((float)x - k.cx) * finvx, zs * ((float)y - k.cy) * finvy, zs);
    s = orc_aff_mul(T, s);
    float u = fmaf(k.fx, s.x / s.z, k.cx);
    float v = fmaf(k.fy, s.y / s.z, k.cy);
    if (s.z <= 0 || u < 0 || v < 0 || u >= (float)cols || v >= (float)rows) return -1;
    if (!(u == u) || !(v == v)) return -1;
    const int dst_z = ((const unsigned short *)((const char *)dprev + (size_t)(int)v * dppitch))[(int)u];
    if (dst_z == 0) return -1;
    const float zd = dst_z * 0.001f;
    orc_f3 d = f3(zd * (u - k.cx) * finvx, zd * (v - k.cy) * finvy, zd);
    orc_f3 df = orc_sub(s, d);
    float dist2 = orc_dot(df, df);
    if (dist2 > dist2_thres) return -1;
    const float *nc = orc_row_f4(ncurr, ncpitch, y) + 4 * x;
    orc_f3 ns = orc_mat_mul(T->R, f3(nc[0], nc[1], nc[2]));
    const float *np = orc_row_f4(nprev, nppitch, (int)v) + 4 * (int)u;
    orc_f3 nd = f3(np[0], np[1], np[2]);
    float cosine = fabsf(orc_dot(ns, nd));
    if (!(cosine >= min_cosine)) { if (cosine < min_cosine) return -1; }   /* NaN cosine passes, as in the reference */
    orc_f3 c = orc_cross(s, nd);
    row[0] = c.x; row[1] = c.y; row[2] = c.z; row[3] = nd.x; row[4] = nd.y; row[5] = nd.z;
    row[6] = orc_dot(nd, orc_sub(d, s));
    return (long long)(int)v * cols + (int)u;
}

/* the 27 products row_i * row_j (i = 0..5, j = i..6) of one row, formed in float (proj_icp.cu:137-345), added to acc in double */
static void icp_add_row(double acc[27], const float row[7])
{
    int shift = 0;
    for (int i = 0; i < 6; ++i)
        for (int j = i; j < 7; ++j) acc[shift++] += (double)(row[i] * row[j]);
}

/* Per-pixel export of the rule: rows7[7 * (y * cols + x)] receives the pixel's row (NaN x 7 when it is rejected), match[y * cols + x]
 * the linear index of the matched previous pixel (-1 when rejected).  An accepted row may itself hold NaN (a NaN previous normal passes
 * the cosine test): match, not the row, tells inliers apart.  Returns the number of inliers. */
long long orc_icp_rows(const float *vcurr, size_t vcpitch, const float *ncurr, size_t ncpitch, const float *vprev, size_t vppitch,
                       const float *nprev, size_t nppitch, int cols, int rows, orc_intr k, orc_aff3f T, float dist2_thres, float min_cosine,
                       float *rows7, int *match)
{
    long long inliers = 0;
    for (int y = 0; y < rows; ++y)
        for (int x = 0; x < cols; ++x) {
            float *row = rows7 + 7 * ((size_t)y * cols + x);
            const long long m = icp_row_points(vcurr, vcpitch, ncurr, ncpitch, vprev, vppitch, nprev, nppitch, cols, rows, k, &T,
                                               dist2_thres, min_cosine, x, y, row);
            if (m < 0) for (int i = 0; i < 7; ++i) row[i] = NAN;
            match[(size_t)y * cols + x] = (int)m;
            inliers += m >= 0;
        }
    return inliers;
}

long long orc_icp_rows_depth(const unsigned short *dcurr, size_t dcpitch, const float *ncurr, size_t ncpitch, const unsigned short *dprev,
                             size_t dppitch, const float *nprev, size_t nppitch, int cols, int rows, orc_intr k, orc_aff3f T,
                             float dist2_thres, float min_cosine, float *rows7, int *match)
{
    long long inliers = 0;
    for (int y = 0; y < rows; ++y)
        for (int x = 0; x < cols; ++x) {
            float *row = rows7 + 7 * ((size_t)y * cols + x);
            const long long m = icp_row_depth(dcurr, dcpitch, ncurr, ncpitch, dprev, dppitch, nprev, nppitch, cols, rows, k, &T,
                                              dist2_thres, min_cosine, x, y, row);
            if (m < 0) for (int i = 0; i < 7; ++i) row[i] = NAN;
            match[(size_t)y * cols + x] = (int)m;
            inliers += m >= 0;
        }
    return inliers;
}

/* The 27 sums of one level: the rows above summed in raster order, in double (the reference's float tree-sum order is launch-geometry
 * dependent).  Returns the number of inlier correspondences. */
long long orc_icp_accumulate(const float *vcurr, size_t vcpitch, const float *ncurr, size_t ncpitch, const float *vprev, size_t vppitch,
                             const float *nprev, size_t nppitch, int cols, int rows, orc_intr k, orc_aff3f T,
                             float dist2_thres, float min_cosine, double *out27)
{
    double acc[27];
    for (int i = 0; i < 27; ++i) acc[i] = 0.0;
    long long inliers = 0;
    for (int y = 0; y < rows; ++y)
        for (int x = 0; x < cols; ++x) {
            float row[7];
            if (icp_row_points(vcurr, vcpitch, ncurr, ncpitch, vprev, vppitch, nprev, nppitch, cols, rows, k, &T, dist2_thres, min_cosine,
                               x, y, row) < 0)
                continue;
            icp_add_row(acc, row);
            ++inliers;
        }
    for (int i = 0; i < 27; ++i) out27[i] = acc[i];
    return inliers;
}

long long orc_icp_accumulate_depth(const unsigned short *dcurr, size_t dcpitch, const float *ncurr, size_t ncpitch, const unsigned short *dprev,
                                   size_t dppitch, const float *nprev, size_t nppitch, int cols, int rows, orc_intr k, orc_aff3f T,
                                   float dist2_thres, float min_cosine, double *out27)
{
    double acc[27];
    for (int i = 0; i < 27; ++i) acc[i] = 0.0;
    long long inliers = 0;
    for (int y = 0; y < rows; ++y)
        for (int x = 0; x < cols; ++x) {
            float row[7];
            if (icp_row_depth(dcurr, dcpitch, ncurr, ncpitch, dprev, dppitch, nprev, nppitch, cols, rows, k, &T, dist2_thres, min_cosine,
                              x, y, row) < 0)
                continue;
            icp_add_row(acc, row);
            ++inliers;
        }
    for (int i = 0; i < 27; ++i) out27[i] = acc[i];
    return inliers;
}

static double det6(const double *Ain)
{
    double A[36];
    memcpy(A, Ain, sizeof A);
    double det = 1.0;
    for (int c = 0; c < 6; ++c) {
        int p = c;
        for (int r = c + 1; r < 6; ++r) if (fabs(A[r * 6 + c]) > fabs(A[p * 6 + c])) p = r;
        if (A[p * 6 + c] == 0.0) return 0.0;
        if (p != c) { for (int j = 0; j < 6; ++j) { double t = A[c * 6 + j]; A[c * 6 + j] = A[p * 6 + j]; A[p * 6 + j] = t; } det = -det; }
        det *= A[c * 6 + c];
        for (int r = c + 1; r < 6; ++r) {
            double f = A[r * 6 + c] / A[c * 6 + c];
            for (int j = c; j < 6; ++j) A[r * 6 + j] -= f * A[c * 6 + j];
        }
    }
    return det;
}

/* symmetric 6x6 solve through cyclic Jacobi eigen-decomposition (== SVD pseudo-inverse for symmetric A) */
static void sym6_solve(const double *Ain, const double *b, double *x)
{
    double A[36], V[36];
    memcpy(A, Ain, sizeof A);
    for (int i = 0; i < 36; ++i) V[i] = 0.0;
    for (int i = 0; i < 6; ++i) V[i * 6 + i] = 1.0;
    for (int sweep = 0; sweep < 60; ++sweep) {
        double off = 0.0;
        for (int p = 0; p < 6; ++p) for (int q = p + 1; q < 6; ++q) off += A[p * 6 + q] * A[p * 6 + q];
        if (off < 1e-300) break;
        for (int p = 0; p < 6; ++p)
            for (int q = p + 1; q < 6; ++q) {
                double apq = A[p * 6 + q];
                if (apq == 0.0) continue;
                double theta = (A[q * 6 + q] - A[p * 6 + p]) / (2.0 * apq);
                double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
                double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
                for (int kx = 0; kx < 6; ++kx) {
                    double akp = A[kx * 6 + p], akq = A[kx * 6 + q];
                    A[kx * 6 + p] = c * akp - s * akq; A[kx * 6 + q] = s * akp + c * akq;
                }
                for (int kx = 0; kx < 6; ++kx) {
                    double apk = A[p * 6 + kx], aqk = A[q * 6 + kx];
                    A[p * 6 + kx] = c * apk - s * aqk; A[q * 6 + kx] = s * apk + c * aqk;
                }
                for (int kx = 0; kx < 6; ++kx) {
                    double vkp = V[kx * 6 + p], vkq = V[kx * 6 + q];
                    V[kx * 6 + p] = c * vkp - s * vkq; V[kx * 6 + q] = s * vkp + c * vkq;
                }
            }
    }
    double wmax = 0.0;
    for (int i = 0; i < 6; ++i) if (fabs(A[i * 6 + i]) > wmax) wmax = fabs(A[i * 6 + i]);
    const double thr = wmax * 6 * DBL_EPSILON;
    for (int i = 0; i < 6; ++i) x[i] = 0.0;
    for (int e = 0; e < 6; ++e) {
        double w = A[e * 6 + e];
        if (fabs(w) <= thr) continue;
        double proj = 0.0;
        for (int i = 0; i < 6; ++i) proj += V[i * 6 + e] * b[i];
        proj /= w;
        for (int i = 0; i < 6; ++i) x[i] += V[i * 6 + e] * proj;
    }
}

/* StreamHelper::get (projective_icp.cpp:43-62) + the per-iteration host step (:195-209):
 * unpack 21+6 sums, det gate, SVD solve, Tinc = Affine3f(rvec = r[0:3], t = r[3:6]), T <- Tinc * T.
 * Returns 0 on the reference's failure path (|det| < 1e-15 or NaN). */
int orc_icp_solve_update(const double *sums27, orc_aff3f *T)
{
    double A[36], b[6];
    int shift = 0;
    for (int i = 0; i < 6; ++i)
        for (int j = i; j < 7; ++j) {
            double value = (double)(float)sums27[shift++];     /* the reference's buffer is float */
            if (j == 6) b[i] = value;
            else A[j * 6 + i] = A[i * 6 + j] = value;
        }
    double det = det6(A);
    if (fabs(det) < 1e-15 || det != det) return 0;
    double r[6];
    sym6_solve(A, b, r);
    float rf[6];
    for (int i = 0; i < 6; ++i) rf[i] = (float)r[i];

    /* cv::Affine3f(rvec, t): Rodrigues in double on float inputs (opencv2/core/affine.hpp) */
    float Rinc[9];
    double theta = sqrt((double)rf[0] * rf[0] + (double)rf[1] * rf[1] + (double)rf[2] * rf[2]);
    if (theta < DBL_EPSILON) {
        for (int i = 0; i < 9; ++i) Rinc[i] = (i % 4 == 0) ? 1.f : 0.f;
    } else {
        double c = cos(theta), s = sin(theta), c1 = 1. - c, itheta = 1. / theta;
        float rx = (float)(rf[0] * itheta), ry = (float)(rf[1] * itheta), rz = (float)(rf[2] * itheta);
        float rrt[9] = {rx * rx, rx * ry, rx * rz, rx * ry, ry * ry, ry * rz, rx * rz, ry * rz, rz * rz};
        float r_x[9] = {0, -rz, ry, rz, 0, -rx, -ry, rx, 0};
        for (int i = 0; i < 9; ++i)
            Rinc[i] = (float)(c * ((i % 4 == 0) ? 1.0 : 0.0) + c1 * rrt[i] + s * r_x[i]);
    }
    /* T <- Tinc * T */
    orc_aff3f out;
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j)
            out.R[i * 3 + j] = Rinc[i * 3 + 0] * T->R[0 * 3 + j] + Rinc[i * 3 + 1] * T->R[1 * 3 + j] + Rinc[i * 3 + 2] * T->R[2 * 3 + j];
        out.t[i] = Rinc[i * 3 + 0] * T->t[0] + Rinc[i * 3 + 1] * T->t[1] + Rinc[i * 3 + 2] * T->t[2] + rf[3 + i];
    }
    *T = out;
    return 1;
}

/* ProjectiveICP::estimateTransform (points variant), projective_icp.cpp:169-213: coarse-to-fine, affine starts
 * at identity, level intrinsics = intr / (1 << level) (setLevelIntr :17-23), min_cosine = cos(angle),
 * dist2 = dist^2 (:11-15). */
int orc_icp_estimate(const float *const *vcurr, const float *const *ncurr, const float *const *vprev, const float *const *nprev,
                     const int *cols, const int *rows, const size_t *pitch, int levels, const int *iters, orc_intr intr,
                     float dist_thres, float angle_thres, orc_aff3f *T_out)
{
    orc_aff3f T;
    for (int i = 0; i < 9; ++i) T.R[i] = (i % 4 == 0) ? 1.f : 0.f;
    T.t[0] = T.t[1] = T.t[2] = 0.f;
    const float min_cosine = cosf(angle_thres);
    const float dist2 = dist_thres * dist_thres;
    for (int level = levels - 1; level >= 0; --level) {
        int div = 1 << level;
        orc_intr k = {intr.fx / div, intr.fy / div, intr.cx / div, intr.cy / div};
        for (int it = 0; it < iters[level]; ++it) {
            double sums[27];
            orc_icp_accumulate(vcurr[level], pitch[level], ncurr[level], pitch[level], vprev[level], pitch[level],
                               nprev[level], pitch[level], cols[level], rows[level], k, T, dist2, min_cosine, sums);
            if (!orc_icp_solve_update(sums, &T)) return 0;
        }
    }
    *T_out = T;
    return 1;
}

/* ProjectiveICP::estimateTransform, depth variant (projective_icp.cpp:126-167): same loop over depth pyramids */
int orc_icp_estimate_depth(const unsigned short *const *dcurr, const float *const *ncurr, const unsigned short *const *dprev,
                           const float *const *nprev, const int *cols, const int *rows, const size_t *dpitch, const size_t *npitch,
                           int levels, const int *iters, orc_intr intr, float dist_thres, float angle_thres, orc_aff3f *T_out)
{
    orc_aff3f T;
    for (int i = 0; i < 9; ++i) T.R[i] = (i % 4 == 0) ? 1.f : 0.f;
    T.t[0] = T.t[1] = T.t[2] = 0.f;
    const float min_cosine = cosf(angle_thres);
    const float dist2 = dist_thres * dist_thres;
    for (int level = levels - 1; level >= 0; --level) {
        int div = 1 << level;
        orc_intr k = {intr.fx / div, intr.fy / div, intr.cx / div, intr.cy / div};
        for (int it = 0; it < iters[level]; ++it) {
            double sums[27];
            orc_icp_accumulate_depth(dcurr[level], dpitch[level], ncurr[level], npitch[level], dprev[level], dpitch[level],
                                     nprev[level], npitch[level], cols[level], rows[level], k, T, dist2, min_cosine, sums);
            if (!orc_icp_solve_update(sums, &T)) return 0;
        }
    }
    *T_out = T;
    return 1;
}
