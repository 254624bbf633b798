/* correspond_oracle.c -- plain C statement of df_mesh_correspond's rule (include/dfusion.h): per pixel of a df_raster_mesh view, the point at
 * the same barycentric position on the source vertex set and the source triangle's face normal; test infrastructure only.  Compiled with
 * -ffp-contract=off so that every float operation is the one the rule names. */
#include <math.h>
#include <stdint.h>
#include <string.h>

#include "oracle_util.h"

/* tri_ids (cols*rows), points (cols*rows*4): a df_raster_mesh result for verts / tris / w12 (world-to-camera, 12 floats); src: the source
 * vertex set (n_verts x vstride); target (cols*rows*4) may be NULL; out_pts, out_nrm: cols*rows*4 floats */
void co_correspond(const int32_t *tri_ids, const float *points, const float *verts, const float *src, int n_verts, int vstride,
                   const int32_t *tris, int n_tris, const float *w12, int cols, int rows, const float *target, float max_dist, float *out_pts,
                   float *out_nrm)
{
    const uint32_t nan_bits = 0x7fffffffu;                  /* the NaN the CUDA kernels write */
    float nanv;
    memcpy(&nanv, &nan_bits, 4);
    const float *R = w12, *t = w12 + 9;
    for (size_t p = 0; p < (size_t)cols * rows; ++p) {
        float *S = out_pts + 4 * p, *N = out_nrm + 4 * p;
        for (int k = 0; k < 4; ++k) S[k] = N[k] = nanv;
        const int id = tri_ids[p];
        if (id < 0 || id >= n_tris) continue;
        const int32_t *ix = tris + 3 * (size_t)id;
        if (ix[0] < 0 || ix[0] >= n_verts || ix[1] < 0 || ix[1] >= n_verts || ix[2] < 0 || ix[2] >= n_verts) continue;
        const float *P = points + 4 * p;
        if (target) {
            const float *T = target + 4 * p;
            if (isnan(T[0]) || isnan(T[1]) || isnan(T[2])) continue;
            const float dx = T[0] - P[0], dy = T[1] - P[1], dz = T[2] - P[2];
            if (dx * dx + dy * dy + dz * dz > max_dist * max_dist) continue;
        }
        float c[3][3];
        const float *s[3];
        for (int k = 0; k < 3; ++k) {
            const float *v = verts + (size_t)ix[k] * vstride;
            const float x = v[0], y = v[1], z = v[2];
            c[k][0] = R[0] * x + R[1] * y + R[2] * z + t[0];
            c[k][1] = R[3] * x + R[4] * y + R[5] * z + t[1];
            c[k][2] = R[6] * x + R[7] * y + R[8] * z + t[2];
            s[k] = src + (size_t)ix[k] * vstride;
        }
        const float e0[3] = {c[1][0] - c[0][0], c[1][1] - c[0][1], c[1][2] - c[0][2]};
        const float e1[3] = {c[2][0] - c[0][0], c[2][1] - c[0][1], c[2][2] - c[0][2]};
        const float q[3] = {P[0] - c[0][0], P[1] - c[0][1], P[2] - c[0][2]};
        const float d00 = dot(e0, e0), d01 = dot(e0, e1), d11 = dot(e1, e1), d20 = dot(q, e0), d21 = dot(q, e1);
        const float den = d00 * d11 - d01 * d01;
        if (!isfinite(den) || den == 0.f) continue;
        const float b1 = (d11 * d20 - d01 * d21) / den, b2 = (d00 * d21 - d01 * d20) / den, b0 = 1.f - b1 - b2;
        for (int k = 0; k < 3; ++k) S[k] = (b0 * s[0][k] + b1 * s[1][k]) + b2 * s[2][k];
        S[3] = 0.f;
        const float a[3] = {s[1][0] - s[0][0], s[1][1] - s[0][1], s[1][2] - s[0][2]};
        const float b[3] = {s[2][0] - s[0][0], s[2][1] - s[0][1], s[2][2] - s[0][2]};
        const float n[3] = {a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]};
        const float len = sqrtf(dot(n, n));
        N[0] = n[0] / len; N[1] = n[1] / len; N[2] = n[2] / len; N[3] = 0.f;
    }
}

/* the barycentric weights of the rule (b0, b1, b2 per pixel, NaN where tri id < 0 or den is not finite or zero); no source, no gate */
void co_weights(const int32_t *tri_ids, const float *points, const float *verts, int vstride, const int32_t *tris, const float *w12, int npix,
                float *b)
{
    const float *R = w12, *t = w12 + 9;
    for (size_t p = 0; p < (size_t)npix; ++p) {
        float *o = b + 3 * p;
        o[0] = o[1] = o[2] = NAN;
        if (tri_ids[p] < 0) continue;
        const int32_t *ix = tris + 3 * (size_t)tri_ids[p];
        float c[3][3];
        for (int k = 0; k < 3; ++k) {
            const float *v = verts + (size_t)ix[k] * vstride;
            const float x = v[0], y = v[1], z = v[2];
            c[k][0] = R[0] * x + R[1] * y + R[2] * z + t[0];
            c[k][1] = R[3] * x + R[4] * y + R[5] * z + t[1];
            c[k][2] = R[6] * x + R[7] * y + R[8] * z + t[2];
        }
        const float *P = points + 4 * p;
        const float e0[3] = {c[1][0] - c[0][0], c[1][1] - c[0][1], c[1][2] - c[0][2]};
        const float e1[3] = {c[2][0] - c[0][0], c[2][1] - c[0][1], c[2][2] - c[0][2]};
        const float q[3] = {P[0] - c[0][0], P[1] - c[0][1], P[2] - c[0][2]};
        const float d00 = dot(e0, e0), d01 = dot(e0, e1), d11 = dot(e1, e1), d20 = dot(q, e0), d21 = dot(q, e1);
        const float den = d00 * d11 - d01 * d01;
        if (!isfinite(den) || den == 0.f) continue;
        o[1] = (d11 * d20 - d01 * d21) / den;
        o[2] = (d00 * d21 - d01 * d20) / den;
        o[0] = 1.f - o[1] - o[2];
    }
}
