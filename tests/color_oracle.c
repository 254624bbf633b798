/* color_oracle.c -- plain C statement of the three colour rules of include/dfusion.h (df_integrate_color, df_sample_colors, df_mesh_colors);
 * test infrastructure only.  Compiled with -ffp-contract=off so that every float operation is the one the rule names; fmaf() only where the
 * rule writes fma. */
#include <math.h>
#include <stdint.h>
#include <string.h>

#include "df_hostmath.h"
#include "oracle_util.h"

/* the rule's constants, restated here rather than taken from dfusion.h so that a change there shows as a disagreement */
#define COLOR_BAND 0.5f
#define ACTIVITY_VOXELS 1024

/* dims, vs, trunc_dist, max_weight: the df_volume's; colors: Dx*Dy*Dz words, updated in place; activity may be NULL; pitches in bytes */
void cl_integrate_color(const int *dims, const float *vs, float trunc_dist, int max_weight, uint32_t *colors, const uint16_t *dists,
                        size_t dists_pitch, const uint8_t *bgra, size_t bgra_pitch, int cols, int rows, const float *vol2cam12,
                        const float *intr4, const uint8_t *activity)
{
    const float *R = vol2cam12, *t = vol2cam12 + 9;
    const float fx = intr4[0], fy = intr4[1], cx = intr4[2], cy = intr4[3];
    const float band = COLOR_BAND * trunc_dist;
    const uint32_t wcap = (uint32_t)(max_weight < 255 ? max_weight : 255);
    size_t i = 0;
    for (int z = 0; z < dims[2]; ++z)
        for (int y = 0; y < dims[1]; ++y)
            for (int x = 0; x < dims[0]; ++x, ++i) {
                if (activity && !activity[i / ACTIVITY_VOXELS]) continue;
                const float p[3] = {(float)x * vs[0], (float)y * vs[1], (float)z * vs[2]};
                float vc[3];
                for (int c = 0; c < 3; ++c) vc[c] = fmaf(R[3 * c], p[0], fmaf(R[3 * c + 1], p[1], R[3 * c + 2] * p[2])) + t[c];
                const float u = fmaf(fx, vc[0] / vc[2], cx), v = fmaf(fy, vc[1] / vc[2], cy);
                if (u < 0 || v < 0 || u >= (float)cols || v >= (float)rows) continue;
                if (vc[2] <= 0) continue;
                if (u != u || v != v) continue;
                const int pu = (int)u, pv = (int)v;
                const float Dp = half_to_float(*(const uint16_t *)((const char *)dists + (size_t)pv * dists_pitch + (size_t)pu * 2));
                if (Dp == 0) continue;
                const float sdf = Dp - sqrtf(fmaf(vc[0], vc[0], fmaf(vc[1], vc[1], vc[2] * vc[2])));
                if (!(fabsf(sdf) <= band)) continue;
                const uint8_t *s = bgra + (size_t)pv * bgra_pitch + (size_t)pu * 4;
                const uint32_t c = colors[i], W = c >> 24, n = W + 1, h = n >> 1;
                const uint32_t r = ((c & 0xffu) * W + s[2] + h) / n, g = (((c >> 8) & 0xffu) * W + s[1] + h) / n,
                               b = (((c >> 16) & 0xffu) * W + s[0] + h) / n;
                colors[i] = r | (g << 8) | (b << 16) | ((n < wcap ? n : wcap) << 24);
            }
}

static uint32_t round_channel(float v)
{
    const int i = (int)rintf(v);                            /* round to nearest, ties to even (the default rounding mode) */
    return (uint32_t)(i < 0 ? 0 : (i > 255 ? 255 : i));
}

/* points: n points of `stride` floats; rgba: n words */
void cl_sample_colors(const int *dims, const float *vs, const uint32_t *colors, const float *vol_pose12, float offset, const float *points,
                      int stride, size_t n, uint32_t *rgba)
{
    float inv[12];
    dfh_aff_inv(vol_pose12, inv);
    const float *R = inv, *t = inv + 9;
    for (size_t q = 0; q < n; ++q) {
        const float *p = points + q * (size_t)stride;
        const float x = p[0], y = p[1], z = p[2];
        rgba[q] = 0;
        if (x != x || y != y || z != z) continue;
        float g[3], fl[3], f[3];
        int ok = 1;
        for (int c = 0; c < 3; ++c) {
            g[c] = (R[3 * c] * x + R[3 * c + 1] * y + R[3 * c + 2] * z + t[c]) / vs[c] - offset;
            if (!(g[c] >= 0.f && g[c] < (float)(dims[c] - 1))) ok = 0;
        }
        if (!ok) continue;
        for (int c = 0; c < 3; ++c) { fl[c] = floorf(g[c]); f[c] = g[c] - fl[c]; }
        const int ix = (int)fl[0], iy = (int)fl[1], iz = (int)fl[2];
        float sw = 0.f, s[3] = {0.f, 0.f, 0.f};
        for (int k = 0; k < 8; ++k) {
            const int dx = k & 1, dy = (k >> 1) & 1, dz = k >> 2;
            const uint32_t c = colors[((size_t)(iz + dz) * dims[1] + (iy + dy)) * dims[0] + (ix + dx)];
            if ((c >> 24) == 0) continue;
            const float wk = ((dx ? f[0] : 1.f - f[0]) * (dy ? f[1] : 1.f - f[1])) * (dz ? f[2] : 1.f - f[2]);
            sw = sw + wk;
            for (int ch = 0; ch < 3; ++ch) s[ch] = s[ch] + wk * (float)((c >> (8 * ch)) & 0xffu);
        }
        if (!(sw > 0.f)) continue;
        rgba[q] = round_channel(s[0] / sw) | (round_channel(s[1] / sw) << 8) | (round_channel(s[2] / sw) << 16) | 0xff000000u;
    }
}

/* tri_ids (npix), points (npix * 4): a df_raster_mesh result for verts / tris / w12; vert_rgba: n_verts words; image: npix * 4 bytes B, G, R, 0.
 * weights (optional, npix * 3): b0, b1, b2 per pixel, NaN where there are none */
void cl_mesh_colors(const int32_t *tri_ids, const float *points, const float *verts, int n_verts, int vstride, const int32_t *tris, int n_tris,
                    const float *w12, const uint32_t *vert_rgba, size_t npix, uint8_t *image, float *weights)
{
    const float *R = w12, *t = w12 + 9;
    for (size_t p = 0; p < npix; ++p) {
        uint8_t *o = image + 4 * p;
        o[0] = o[1] = o[2] = o[3] = 0;
        if (weights) weights[3 * p] = weights[3 * p + 1] = weights[3 * p + 2] = NAN;
        const int id = tri_ids[p];
        if (id < 0 || id >= n_tris) continue;
        const int32_t *ix = tris + 3 * (size_t)id;
        if (ix[0] < 0 || ix[0] >= n_verts || ix[1] < 0 || ix[1] >= n_verts || ix[2] < 0 || ix[2] >= n_verts) continue;
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
        float b[3];
        b[1] = (d11 * d20 - d01 * d21) / den;
        b[2] = (d00 * d21 - d01 * d20) / den;
        b[0] = 1.f - b[1] - b[2];
        if (weights) memcpy(weights + 3 * p, b, 12);
        float sw = 0.f, s[3] = {0.f, 0.f, 0.f};
        for (int k = 0; k < 3; ++k) {
            const uint32_t col = vert_rgba[ix[k]];
            if ((col >> 24) == 0) continue;
            sw = sw + b[k];
            for (int ch = 0; ch < 3; ++ch) s[ch] = s[ch] + b[k] * (float)((col >> (8 * ch)) & 0xffu);
        }
        if (!(sw > 0.f)) continue;
        o[0] = (uint8_t)round_channel(s[2] / sw);
        o[1] = (uint8_t)round_channel(s[1] / sw);
        o[2] = (uint8_t)round_channel(s[0] / sw);
    }
}

void cl_aff_mul(const float *a, const float *b, float *out) { dfh_aff_mul(a, b, out); }
void cl_aff_inv(const float *a, float *out) { dfh_aff_inv(a, out); }
