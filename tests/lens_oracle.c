/* lens_oracle.c -- plain C statement of the lens rules of include/dfusion.h: the distortion of df_lens, df_undistort, and the colour
 * camera's projection through its lens in df_color_depth_map_lens, df_integrate_color_camera_lens and df_frame_intensity_lens; test
 * infrastructure only.  It includes color_camera_oracle.c for the colour-camera rules' shared pieces (the cell rule, the pinhole projection a
 * NULL lens takes, and through it oracle_util.h's affine and fp16 helpers).  Compiled with -ffp-contract=off so that every float operation
 * is the one the rule names; fmaf() only where the rule writes fma. */
#include "color_camera_oracle.c"

/* lens: k1, k2, p1, p2, k3, k4, k5, k6, r2_max (df_lens' field order); returns 0 when (x, y) is outside the calibrated radius or NaN */
int lens_distort(const float *L, float x, float y, float *xd, float *yd)
{
    const float r2 = x * x + y * y;
    if (!(r2 <= L[8])) return 0;
    const float radial = (1.f + r2 * (L[0] + r2 * (L[1] + r2 * L[4]))) / (1.f + r2 * (L[5] + r2 * (L[6] + r2 * L[7])));
    *xd = x * radial + (2.f * L[2] * x * y + L[3] * (r2 + 2.f * x * x));
    *yd = y * radial + (L[2] * (r2 + 2.f * y * y) + 2.f * L[3] * x * y);
    return 1;
}

static int lens_is_zero(const float *L)
{
    for (int i = 0; i < 8; ++i)
        if (L[i] != 0.f) return 0;
    return 1;
}

/* df_undistort: depth / out u16, bgra / bout 4 bytes per pixel (both NULL without colour); pitches in bytes */
void lens_undistort(const uint16_t *depth, size_t dpitch, uint16_t *out, size_t opitch, const uint8_t *bgra, size_t bpitch, uint8_t *bout,
                    size_t bopitch, int cols, int rows, const float *intr4, const float *lens)
{
    float L[9];
    memcpy(L, lens, sizeof L);
    if (lens_is_zero(L)) L[8] = INFINITY;
    const float fx = intr4[0], fy = intr4[1], cx = intr4[2], cy = intr4[3], finvx = 1.f / fx, finvy = 1.f / fy;
    for (int j = 0; j < rows; ++j)
        for (int i = 0; i < cols; ++i) {
            const float x = ((float)i - cx) * finvx, y = ((float)j - cy) * finvy;
            uint16_t d = 0;
            uint8_t c[4] = {0, 0, 0, 0};
            float xd, yd;
            if (lens_distort(L, x, y, &xd, &yd)) {
                const float su = floorf(fmaf(fx, xd, cx) + 0.5f), sv = floorf(fmaf(fy, yd, cy) + 0.5f);
                if (su >= 0.f && sv >= 0.f && su < (float)cols && sv < (float)rows) {
                    d = *(const uint16_t *)((const char *)depth + (size_t)sv * dpitch + (size_t)su * 2);
                    if (bgra) memcpy(c, bgra + (size_t)sv * bpitch + (size_t)su * 4, 4);
                }
            }
            *(uint16_t *)((char *)out + (size_t)j * opitch + (size_t)i * 2) = d;
            if (bgra) memcpy(bout + (size_t)j * bopitch + (size_t)i * 4, c, 4);
        }
}

/* the colour pixel of pc through the lens (NULL: color_camera_oracle.c's pinhole projection) */
static int project_lens(const float *pc, const float *cam4, const float *lens, int ccols, int crows, float *u, float *v)
{
    if (!lens) return project_color(pc, cam4, ccols, crows, u, v);
    float xd, yd;
    if (!lens_distort(lens, pc[0] / pc[2], pc[1] / pc[2], &xd, &yd)) return 0;
    *u = fmaf(cam4[0], xd, cam4[2]);
    *v = fmaf(cam4[1], yd, cam4[3]);
    if (!(pc[2] > 0)) return 0;
    if (*u != *u || *v != *v) return 0;
    return *u >= 0 && *v >= 0 && *u < (float)ccols && *v < (float)crows;
}

/* df_color_depth_map_lens: cc_depth_map's arguments and the lens (NULL or the zero lens: the pinhole rule) */
void lens_depth_map(const uint16_t *depth, size_t depth_pitch, int cols, int rows, const float *intr4, int ccols, int crows, const float *cam4,
                    const float *d2c12, const float *lens, uint32_t *map, size_t map_pitch)
{
    if (lens && lens_is_zero(lens)) lens = NULL;
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
            if (!project_lens(pc, cam4, lens, ccols, crows, &u, &v)) continue;
            uint32_t *w = (uint32_t *)((char *)map + (size_t)((int)v / cell) * map_pitch + (size_t)((int)u / cell) * 4);
            const uint32_t b = float_bits(pc[2]);
            if (b < *w) *w = b;
        }
}

/* the colour camera's sample of the depth-frame point p: projection through the lens, then the occlusion test; 0 where it does not see p */
static int camera_sample(const float *p, const float *cam4, const float *d2c12, const float *lens, int ccols, int crows, int cell, const uint32_t *map,
                         size_t map_pitch, float tol, const uint8_t *bgra, size_t bgra_pitch, const uint8_t **s)
{
    float pc[3], uc, vcc;
    aff_apply(d2c12, p, pc);
    if (!project_lens(pc, cam4, lens, ccols, crows, &uc, &vcc)) return 0;
    const int iu = (int)uc, iv = (int)vcc;
    const uint32_t zmin = *(const uint32_t *)((const char *)map + (size_t)(iv / cell) * map_pitch + (size_t)(iu / cell) * 4);
    if (zmin == MAP_EMPTY) return 0;
    if (pc[2] > bits_float(zmin) + tol) return 0;
    *s = bgra + (size_t)iv * bgra_pitch + (size_t)iu * 4;
    return 1;
}

/* df_integrate_color_camera_lens: cc_integrate_color_camera's arguments and the lens */
void lens_integrate_color_camera(const int *dims, const float *vs, float trunc_dist, int max_weight, uint32_t *colors, const uint16_t *dists,
                                 size_t dists_pitch, int cols, int rows, const float *vol2cam12, const float *intr4, int ccols, int crows,
                                 const float *cam4, const float *d2c12, const float *lens, const uint8_t *bgra, size_t bgra_pitch,
                                 const uint32_t *map, size_t map_pitch, const uint8_t *activity)
{
    if (lens && lens_is_zero(lens)) lens = NULL;
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
                const float u = fmaf(fx, vc[0] / vc[2], cx), v = fmaf(fy, vc[1] / vc[2], cy);
                if (u < 0 || v < 0 || u >= (float)cols || v >= (float)rows) continue;
                if (vc[2] <= 0) continue;
                if (u != u || v != v) continue;
                const float Dp = half_to_float(*(const uint16_t *)((const char *)dists + (size_t)(int)v * dists_pitch + (size_t)(int)u * 2));
                if (Dp == 0) continue;
                const float sdf = Dp - sqrtf(fmaf(vc[0], vc[0], fmaf(vc[1], vc[1], vc[2] * vc[2])));
                if (!(fabsf(sdf) <= band)) continue;
                const uint8_t *s;
                if (!camera_sample(vc, cam4, d2c12, lens, ccols, crows, cell, map, map_pitch, tol, bgra, bgra_pitch, &s)) continue;
                const uint32_t c = colors[i], W = c >> 24, n = W + 1, h = n >> 1;
                const uint32_t r = ((c & 0xffu) * W + s[2] + h) / n, g = (((c >> 8) & 0xffu) * W + s[1] + h) / n,
                               b = (((c >> 16) & 0xffu) * W + s[0] + h) / n;
                colors[i] = r | (g << 8) | (b << 16) | ((n < wcap ? n : wcap) << 24);
            }
}

/* level 0 of df_frame_intensity_lens through a colour camera: points dense float4 cols x rows; out dense floats (NaN = no value) */
void lens_frame_intensity(const uint8_t *bgra, size_t bgra_pitch, int ccols, int crows, const float *cam4, const float *d2c12, const float *lens,
                          const float *intr4, const uint32_t *map, size_t map_pitch, float trunc_dist, const float *points, int cols, int rows,
                          float *out)
{
    if (lens && lens_is_zero(lens)) lens = NULL;
    const int cell = cc_cell(intr4, cam4);
    const float tol = COLOR_OCCLUSION * trunc_dist;
    for (int y = 0; y < rows; ++y)
        for (int x = 0; x < cols; ++x) {
            const float *p = points + ((size_t)y * cols + x) * 4;
            const uint8_t *s;
            float I = NAN;
            if (!isnan(p[0]) && camera_sample(p, cam4, d2c12, lens, ccols, crows, cell, map, map_pitch, tol, bgra, bgra_pitch, &s))
                I = (float)((77u * s[2] + 150u * s[1] + 29u * s[0] + 128u) >> 8) / 255.f;
            out[(size_t)y * cols + x] = I;
        }
}
