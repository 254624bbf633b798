/* color_track_oracle.c -- plain-C restatement of the colour-tracking rules of include/dfusion.h (df_frame_intensity, df_model_intensity and
 * the photometric row of df_icp_accumulate_color), operation for operation, for bit-exact comparison with csrc/color.cu and csrc/icp.cu.
 * Built with -ffp-contract=off: float operations are IEEE round-to-nearest, fmaf only where the rules write fma. */
#include <math.h>
#include <stddef.h>
#include <stdint.h>
#include <string.h>

#include "oracle_util.h"

static float luma(uint32_t r, uint32_t g, uint32_t b) { return (float)((77u * r + 150u * g + 29u * b + 128u) >> 8) / 255.f; }

/* level 0, registered image: out[y * cols + x] = intensity of bgra pixel (x, y) */
void ct_intensity_registered(const uint8_t *bgra, size_t pitch, int cols, int rows, float *out)
{
    for (int y = 0; y < rows; ++y)
        for (int x = 0; x < cols; ++x) {
            const uint8_t *c = bgra + (size_t)y * pitch + (size_t)x * 4;
            out[(size_t)y * cols + x] = luma(c[2], c[1], c[0]);
        }
}

/* level 0 through a colour camera: points dense float4 cols x rows; cam4 = colour (fx, fy, cx, cy), ccols x crows; d2c12 depth_to_color;
 * map: df_color_depth_map's words, mcols per row (pitch in bytes), cell; tol = DF_COLOR_OCCLUSION * trunc_dist as one float product */
void ct_intensity_camera(const uint8_t *bgra, size_t bpitch, int ccols, int crows, const float *cam4, const float *d2c12, int cell, const uint32_t *map,
                         size_t mpitch, float occlusion, float trunc_dist, const float *points, int cols, int rows, float *out)
{
    const float tol = occlusion * trunc_dist;
    for (int y = 0; y < rows; ++y)
        for (int x = 0; x < cols; ++x) {
            const float *p = points + ((size_t)y * cols + x) * 4;
            float I = NAN;
            if (!isnan(p[0])) {
                float pc[3];
                aff_apply(d2c12, p, pc);
                const float u = fmaf(cam4[0], pc[0] / pc[2], cam4[2]), v = fmaf(cam4[1], pc[1] / pc[2], cam4[3]);
                if (pc[2] > 0 && u >= 0 && v >= 0 && u < (float)ccols && v < (float)crows) {
                    const int iu = (int)u, iv = (int)v;
                    const uint32_t zw = *(const uint32_t *)((const char *)map + (size_t)(iv / cell) * mpitch + (size_t)(iu / cell) * 4);
                    float zmin;
                    memcpy(&zmin, &zw, 4);
                    if (zw != 0xffffffffu && !(pc[2] > zmin + tol)) {
                        const uint8_t *c = bgra + (size_t)iv * bpitch + (size_t)iu * 4;
                        I = luma(c[2], c[1], c[0]);
                    }
                }
            }
            out[(size_t)y * cols + x] = I;
        }
}

/* level l from level l - 1 (src: scols per row, dense): the mean of the valid values of each 2 x 2 block, (0,0), (1,0), (0,1), (1,1) */
void ct_intensity_down(const float *src, int scols, float *dst, int cols, int rows)
{
    for (int y = 0; y < rows; ++y)
        for (int x = 0; x < cols; ++x) {
            float s = 0.f;
            int n = 0;
            for (int dy = 0; dy < 2; ++dy)
                for (int dx = 0; dx < 2; ++dx) {
                    const float v = src[(size_t)(2 * y + dy) * scols + 2 * x + dx];
                    if (!isnan(v)) { s = s + v; ++n; }
                }
            dst[(size_t)y * cols + x] = n ? s / (float)n : NAN;
        }
}

/* df_sample_colors' rule with the transform a12 applied as written (r.x*x + r.y*y + r.z*z + t, left to right) and offset 0 */
static uint32_t sample(const int *dims, const float *vs, const uint32_t *colors, const float *a12, const float *p)
{
    const float x = p[0], y = p[1], z = p[2];
    if (x != x || y != y || z != z) return 0u;
    const float g[3] = {(a12[0] * x + a12[1] * y + a12[2] * z + a12[9]) / vs[0] - 0.f, (a12[3] * x + a12[4] * y + a12[5] * z + a12[10]) / vs[1] - 0.f,
                        (a12[6] * x + a12[7] * y + a12[8] * z + a12[11]) / vs[2] - 0.f};
    for (int c = 0; c < 3; ++c)
        if (!(g[c] >= 0.f && g[c] < (float)(dims[c] - 1))) return 0u;
    const float fl[3] = {floorf(g[0]), floorf(g[1]), floorf(g[2])};
    const int ix = (int)fl[0], iy = (int)fl[1], iz = (int)fl[2];
    const float f[3] = {g[0] - fl[0], g[1] - fl[1], g[2] - fl[2]};
    const float wx[2] = {1.f - f[0], f[0]}, wy[2] = {1.f - f[1], f[1]}, wz[2] = {1.f - f[2], f[2]};
    float sw = 0.f, sr = 0.f, sg = 0.f, sb = 0.f;
    for (int k = 0; k < 8; ++k) {
        const int dx = k & 1, dy = (k >> 1) & 1, dz = k >> 2;
        const uint32_t c = colors[((size_t)(iz + dz) * dims[1] + (iy + dy)) * dims[0] + (ix + dx)];
        if ((c >> 24) == 0) continue;
        const float wk = (wx[dx] * wy[dy]) * wz[dz];
        sw = sw + wk;
        sr = sr + wk * (float)(c & 0xffu);
        sg = sg + wk * (float)((c >> 8) & 0xffu);
        sb = sb + wk * (float)((c >> 16) & 0xffu);
    }
    if (!(sw > 0.f)) return 0u;
    float ch[3] = {rintf(sr / sw), rintf(sg / sw), rintf(sb / sw)};
    uint32_t out = 0xff000000u;
    for (int c = 0; c < 3; ++c) out |= (uint32_t)(ch[c] > 255.f ? 255 : (int)ch[c]) << (8 * c);
    return out;
}

/* df_model_intensity of one level: points dense float4 cols x rows (camera frame), out dense float4 (I, gu, gv, 0) or four NaNs */
void ct_model_intensity(const int *dims, const float *vs, const uint32_t *colors, const float *cam2vol12, const float *points, int cols, int rows,
                        float *out, float *I)
{
    for (int i = 0; i < cols * rows; ++i) {
        const uint32_t c = sample(dims, vs, colors, cam2vol12, points + (size_t)i * 4);
        I[i] = c ? luma(c & 0xffu, (c >> 8) & 0xffu, (c >> 16) & 0xffu) : NAN;
    }
    for (int y = 0; y < rows; ++y)
        for (int x = 0; x < cols; ++x) {
            float *o = out + ((size_t)y * cols + x) * 4;
            o[0] = o[1] = o[2] = o[3] = NAN;
            if (x == 0 || y == 0 || x == cols - 1 || y == rows - 1) continue;
            const float c = I[(size_t)y * cols + x];
            const float gu = (I[(size_t)y * cols + x + 1] - I[(size_t)y * cols + x - 1]) * 0.5f;
            const float gv = (I[(size_t)(y + 1) * cols + x] - I[(size_t)(y - 1) * cols + x]) * 0.5f;
            if (isnan(c) || isnan(gu) || isnan(gv)) continue;
            o[0] = c; o[1] = gu; o[2] = gv; o[3] = 0.f;
        }
}

/* the photometric rows of one level: for every pixel whose geometric row exists (match >= 0, the oracle's orc_icp_rows), s = T * v_curr and
 * (u, v) as the geometric rule forms them, then the photometric rule.  rows7: 7 floats per pixel (NaN where there is no row).  Returns the
 * number of rows. */
long ct_photo_rows(const float *vcurr, const float *icurr, const float *model, const int32_t *match, int cols, int rows, const float *K4,
                   const float *T12, float weight, float max_residual, float *rows7)
{
    long n = 0;
    for (int y = 0; y < rows; ++y)
        for (int x = 0; x < cols; ++x) {
            const size_t i = (size_t)y * cols + x;
            float *row = rows7 + i * 7;
            for (int k = 0; k < 7; ++k) row[k] = NAN;
            if (match[i] < 0) continue;
            const float ic = icurr[i];
            if (isnan(ic)) continue;
            float s[3];
            aff_apply(T12, vcurr + i * 4, s);
            const float u = fmaf(K4[0], s[0] / s[2], K4[2]), v = fmaf(K4[1], s[1] / s[2], K4[3]);
            const float fu = floorf(u), fv = floorf(v);
            const int i0 = (int)fu, j0 = (int)fv;
            if (i0 + 1 >= cols || j0 + 1 >= rows) continue;
            const float *m00 = model + ((size_t)j0 * cols + i0) * 4, *m10 = m00 + 4, *m01 = model + ((size_t)(j0 + 1) * cols + i0) * 4, *m11 = m01 + 4;
            if (isnan(m00[0]) || isnan(m10[0]) || isnan(m01[0]) || isnan(m11[0])) continue;
            const float a = u - fu, b = v - fv, a1 = 1.f - a, b1 = 1.f - b;
            float val[3];
            for (int c = 0; c < 3; ++c) val[c] = (m00[c] * a1 + m10[c] * a) * b1 + (m01[c] * a1 + m11[c] * a) * b;
            const float r = ic - val[0];
            if (fabsf(r) > max_residual) continue;
            const float gfx = val[1] * K4[0], gfy = val[2] * K4[1];
            const float g[3] = {gfx / s[2], gfy / s[2], -(gfx * s[0] + gfy * s[1]) / (s[2] * s[2])};
            const float cr[3] = {s[1] * g[2] - s[2] * g[1], s[2] * g[0] - s[0] * g[2], s[0] * g[1] - s[1] * g[0]};
            row[0] = weight * cr[0]; row[1] = weight * cr[1]; row[2] = weight * cr[2];
            row[3] = weight * g[0]; row[4] = weight * g[1]; row[5] = weight * g[2];
            row[6] = weight * r;
            ++n;
        }
    return n;
}
