/* warped_color_oracle.c -- plain C statement of df_integrate_warped_color's colour rule (include/dfusion.h); test infrastructure only.
 *
 * The rule reads values the warped fusion forms per voxel (the warped camera-frame point, its depth pixel and rho), and both halves are
 * already stated once: the warp and the TSDF update in oracle/orc_fusion.c, the colour camera's projection, lens and occlusion test in
 * lens_oracle.c (over color_camera_oracle.c).  Neither is restated here.  orc_fusion.c is compiled into this library unchanged, with one
 * hook: its TSDF store `*vptr = orc_pack_tsdf(...)`, which runs exactly for the voxels the rule writes, first records that voxel's
 * (tx, ty, tz, u, v, rho).  Its warp calls (orc_knn8_fast, orc_dqb, orc_dq_transform) and orc_half2float are liborc.so's: load that
 * library with RTLD_GLOBAL before this one.  wc_fuse then applies the band, the sample and the running average to the records.
 * Compiled with -ffp-contract=off so that every float operation is the one the rule names; fmaf() only where the rule writes fma. */
#include "../oracle/orc_common.h"
#include "lens_oracle.c"

static float *wc_rec;           /* per voxel: tx, ty, tz, u, v, rho of the voxel's TSDF update */
static uint8_t *wc_hit;         /* per voxel: 1 where the TSDF side wrote it */

static void wc_note(size_t i, float tx, float ty, float tz, float u, float v, float rho)
{
    float *r = wc_rec + i * 6;
    r[0] = tx; r[1] = ty; r[2] = tz; r[3] = u; r[4] = v; r[5] = rho;
    wc_hit[i] = 1;
}

/* the hook (a function-like macro is not expanded again inside its own replacement, so the store itself is unchanged), and the two entries
 * of orc_fusion.c under names of their own, so that this library does not export liborc.so's */
#define orc_pack_tsdf(tsdf, weight) (wc_note((size_t)(vptr - vol.data), tx, ty, tz, u, v, rho), orc_pack_tsdf(tsdf, weight))
#define orc_integrate_warped wc_integrate_warped
#define orc_extend_field wc_extend_field_unused
#include "../oracle/orc_fusion.c"
#undef orc_pack_tsdf
#undef orc_integrate_warped
#undef orc_extend_field

/* orc_integrate_warped's arguments (the volume updated in place, its return value) and the records: rec [Dx*Dy*Dz*6] floats, hit
 * [Dx*Dy*Dz] bytes, both zeroed by the caller */
long long wc_integrate_warped_records(orc_volume vol, const uint16_t *depth, size_t pitch, int cols, int rows, orc_aff3f vol2world,
                                      orc_aff3f world2cam, orc_intr intr, const float *nodes, int M, float weight_scale, float *rec, uint8_t *hit)
{
    wc_rec = rec; wc_hit = hit;
    const long long n = wc_integrate_warped(vol, depth, pitch, cols, rows, vol2world, world2cam, intr, nodes, M, weight_scale);
    wc_rec = NULL; wc_hit = NULL;
    return n;
}

/* df_integrate_warped_color's colour side over the records: colors (nvox words) updated in place; returns the voxels coloured.
 * cam4 == NULL: bgra is registered to the depth; else the colour camera (ccols x crows, cam4, d2c12, lens: NULL or 9 floats, map as
 * lens_depth_map writes it) with intr4 the depth intrinsics (for the map's cell). */
long long wc_fuse(long long nvox, const float *rec, const uint8_t *hit, float trunc_dist, int max_weight, uint32_t *colors, const uint8_t *bgra,
                  size_t bgra_pitch, const float *intr4, int ccols, int crows, const float *cam4, const float *d2c12, const float *lens,
                  const uint32_t *map, size_t map_pitch)
{
    if (lens && lens_is_zero(lens)) lens = NULL;
    const float band = COLOR_BAND * trunc_dist, tol = COLOR_OCCLUSION * trunc_dist;
    const int cell = cam4 ? cc_cell(intr4, cam4) : 1;
    const uint32_t wcap = (uint32_t)(max_weight < 255 ? max_weight : 255);
    long long n_col = 0;
    for (long long i = 0; i < nvox; ++i) {
        if (!hit[i]) continue;
        const float *r = rec + i * 6;
        if (!(fabsf(r[5]) <= band)) continue;
        const uint8_t *s;
        if (!cam4) s = bgra + (size_t)(int)r[4] * bgra_pitch + (size_t)(int)r[3] * 4;
        else if (!camera_sample(r, cam4, d2c12, lens, ccols, crows, cell, map, map_pitch, tol, bgra, bgra_pitch, &s)) continue;
        const uint32_t c = colors[i], W = c >> 24, n = W + 1, h = n >> 1;
        const uint32_t cr = ((c & 0xffu) * W + s[2] + h) / n, cg = (((c >> 8) & 0xffu) * W + s[1] + h) / n,
                       cb = (((c >> 16) & 0xffu) * W + s[0] + h) / n;
        colors[i] = cr | (cg << 8) | (cb << 16) | ((n < wcap ? n : wcap) << 24);
        ++n_col;
    }
    return n_col;
}
