/* color_camera_oracle.c -- plain C statement of the two colour-camera rules of include/dfusion.h (df_color_depth_map and
 * df_integrate_color_camera, with df_color_map_dims' cell rule); test infrastructure only.  Compiled with -ffp-contract=off so that every
 * float operation is the one the rule names; fmaf() only where the rule writes fma. */
#include <math.h>
#include <stdint.h>
#include <string.h>

#include "oracle_util.h"

/* the rule's constants, restated here rather than taken from dfusion.h so that a change there shows as a disagreement */
#define COLOR_BAND 0.5f
#define COLOR_OCCLUSION 1.0f
#define ACTIVITY_VOXELS 1024
#define MAP_EMPTY 0xffffffffu

/* cam4: colour fx, fy, cx, cy; returns 1 and the colour pixel (u, v) when pc lies in front of the colour camera and inside its image */
static int project_color(const float *pc, const float *cam4, int ccols, int crows, float *u, float *v)
{
    *u = fmaf(cam4[0], pc[0] / pc[2], cam4[2]);
    *v = fmaf(cam4[1], pc[1] / pc[2], cam4[3]);
    if (!(pc[2] > 0)) return 0;
    if (*u != *u || *v != *v) return 0;
    return *u >= 0 && *v >= 0 && *u < (float)ccols && *v < (float)crows;
}

/* df_color_map_dims' cell rule */
int cc_cell(const float *intr4, const float *cam4)
{
    const int c = (int)ceilf(fmaxf(cam4[0] / intr4[0], cam4[1] / intr4[1]));
    return c > 1 ? c : 1;
}

/* depth: rows x cols u16 (pitch in bytes); map: ceil(ccols / cell) x ceil(crows / cell) words, pitch in bytes, overwritten */
void cc_depth_map(const uint16_t *depth, size_t depth_pitch, int cols, int rows, const float *intr4, int ccols, int crows, const float *cam4,
                  const float *d2c12, uint32_t *map, size_t map_pitch)
{
    const int cell = cc_cell(intr4, cam4), mcols = (ccols + cell - 1) / cell, mrows = (crows + cell - 1) / cell;
    for (int r = 0; r < mrows; ++r)
        for (int c = 0; c < mcols; ++c) *(uint32_t *)((char *)map + (size_t)r * map_pitch + (size_t)c * 4) = MAP_EMPTY;
    const float finvx = 1.f / intr4[0], finvy = 1.f / intr4[1], cx = intr4[2], cy = intr4[3];
    for (int j = 0; j < rows; ++j)
        for (int i = 0; i < cols; ++i) {
            const uint16_t d = *(const uint16_t *)((const char *)depth + (size_t)j * depth_pitch + (size_t)i * 2);
            if (d == 0) continue;
            const float z = (float)d * 0.001f;
            const float p[3] = {z * ((float)i - cx) * finvx, z * ((float)j - cy) * finvy, z};
            float pc[3], u, v;
            aff_apply(d2c12, p, pc);
            if (!project_color(pc, cam4, ccols, crows, &u, &v)) continue;
            uint32_t *w = (uint32_t *)((char *)map + (size_t)((int)v / cell) * map_pitch + (size_t)((int)u / cell) * 4);
            const uint32_t b = float_bits(pc[2]);
            if (b < *w) *w = b;
        }
}

/* df_integrate_color_camera: dims, vs, trunc_dist, max_weight: the df_volume's; colors updated in place; dists: the depth frame's (cols x
 * rows); bgra: the colour image (ccols x crows); map as cc_depth_map writes it; activity may be NULL; pitches in bytes */
void cc_integrate_color_camera(const int *dims, const float *vs, float trunc_dist, int max_weight, uint32_t *colors, const uint16_t *dists,
                               size_t dists_pitch, int cols, int rows, const float *vol2cam12, const float *intr4, int ccols, int crows,
                               const float *cam4, const float *d2c12, const uint8_t *bgra, size_t bgra_pitch, const uint32_t *map,
                               size_t map_pitch, const uint8_t *activity)
{
    const float fx = intr4[0], fy = intr4[1], cx = intr4[2], cy = intr4[3];
    const float band = COLOR_BAND * trunc_dist, tol = COLOR_OCCLUSION * trunc_dist;
    const int cell = cc_cell(intr4, cam4);
    const uint32_t wcap = (uint32_t)(max_weight < 255 ? max_weight : 255);
    size_t i = 0;
    for (int z = 0; z < dims[2]; ++z)
        for (int y = 0; y < dims[1]; ++y)
            for (int x = 0; x < dims[0]; ++x, ++i) {
                if (activity && !activity[i / ACTIVITY_VOXELS]) continue;
                const float p[3] = {(float)x * vs[0], (float)y * vs[1], (float)z * vs[2]};
                float vc[3];
                aff_apply(vol2cam12, p, vc);
                /* the depth side: df_integrate_color's tests, in its order */
                const float u = fmaf(fx, vc[0] / vc[2], cx), v = fmaf(fy, vc[1] / vc[2], cy);
                if (u < 0 || v < 0 || u >= (float)cols || v >= (float)rows) continue;
                if (vc[2] <= 0) continue;
                if (u != u || v != v) continue;
                const float Dp = half_to_float(*(const uint16_t *)((const char *)dists + (size_t)(int)v * dists_pitch + (size_t)(int)u * 2));
                if (Dp == 0) continue;
                const float sdf = Dp - sqrtf(fmaf(vc[0], vc[0], fmaf(vc[1], vc[1], vc[2] * vc[2])));
                if (!(fabsf(sdf) <= band)) continue;
                /* the colour camera: projection, then occlusion */
                float pc[3], uc, vcc;
                aff_apply(d2c12, vc, pc);
                if (!project_color(pc, cam4, ccols, crows, &uc, &vcc)) continue;
                const int iu = (int)uc, iv = (int)vcc;
                const uint32_t zmin = *(const uint32_t *)((const char *)map + (size_t)(iv / cell) * map_pitch + (size_t)(iu / cell) * 4);
                if (zmin == MAP_EMPTY) continue;
                if (pc[2] > bits_float(zmin) + tol) continue;
                const uint8_t *s = bgra + (size_t)iv * bgra_pitch + (size_t)iu * 4;
                const uint32_t c = colors[i], W = c >> 24, n = W + 1, h = n >> 1;
                const uint32_t r = ((c & 0xffu) * W + s[2] + h) / n, g = (((c >> 8) & 0xffu) * W + s[1] + h) / n,
                               b = (((c >> 16) & 0xffu) * W + s[0] + h) / n;
                colors[i] = r | (g << 8) | (b << 16) | ((n < wcap ? n : wcap) << 24);
            }
}
