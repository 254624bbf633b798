// color_sample.cuh -- the colour rules of include/dfusion.h that more than one kernel states, written once: the colour volume's sample at a
// point (df_sample_colors' rule: df_sample_colors and df_model_intensity, csrc/color.cu), and the fusion side's integer running average and
// colour-camera projection with its occlusion test (df_integrate_color, df_integrate_color_camera and df_frame_intensity in csrc/color.cu;
// df_integrate_warped_color in csrc/fusion.cu).
#pragma once
#include "df_common.cuh"
#include "lens.cuh"

namespace dfb {

struct SampleParams {
    const uint32_t *colors;
    int Dx, Dy, Dz;
    float vsx, vsy, vsz, offset;
    Aff world2vol;
    const char *points; size_t ppitch; int stride;
    int cols, rows;
    const int *count;
    char *rgba; size_t opitch;
};

__device__ __forceinline__ uint32_t sample_color(const SampleParams &p, float x, float y, float z)
{
    if (x != x || y != y || z != z) return 0u;
    const Aff &a = p.world2vol;
    const float gx = (a.r0.x * x + a.r0.y * y + a.r0.z * z + a.t.x) / p.vsx - p.offset;
    const float gy = (a.r1.x * x + a.r1.y * y + a.r1.z * z + a.t.y) / p.vsy - p.offset;
    const float gz = (a.r2.x * x + a.r2.y * y + a.r2.z * z + a.t.z) / p.vsz - p.offset;
    if (!(gx >= 0.f && gx < (float)(p.Dx - 1) && gy >= 0.f && gy < (float)(p.Dy - 1) && gz >= 0.f && gz < (float)(p.Dz - 1))) return 0u;
    const float flx = floorf(gx), fly = floorf(gy), flz = floorf(gz);
    const int ix = (int)flx, iy = (int)fly, iz = (int)flz;
    const float fx = gx - flx, fy = gy - fly, fz = gz - flz;
    const float wx[2] = {1.f - fx, fx}, wy[2] = {1.f - fy, fy}, wz[2] = {1.f - fz, fz};
    float sw = 0.f, sr = 0.f, sg = 0.f, sb = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const int dx = k & 1, dy = (k >> 1) & 1, dz = k >> 2;
        const uint32_t c = __ldg(p.colors + ((size_t)(iz + dz) * p.Dy + (iy + dy)) * p.Dx + (ix + dx));
        if ((c >> 24) == 0) continue;
        const float wk = (wx[dx] * wy[dy]) * wz[dz];
        sw = sw + wk;
        sr = sr + wk * (float)(c & 0xffu);
        sg = sg + wk * (float)((c >> 8) & 0xffu);
        sb = sb + wk * (float)((c >> 16) & 0xffu);
    }
    if (!(sw > 0.f)) return 0u;
    const uint32_t r = (uint32_t)min(__float2int_rn(sr / sw), 255), g = (uint32_t)min(__float2int_rn(sg / sw), 255),
                   b = (uint32_t)min(__float2int_rn(sb / sw), 255);
    return r | (g << 8) | (b << 16) | 0xff000000u;
}

// integer running average of one voxel word (R, G, B, W) with the sample s (B, G, R, x)
__device__ __forceinline__ uint32_t color_update(uint32_t c, uchar4 s, int wcap)
{
    const uint32_t W = c >> 24, n = W + 1, h = n >> 1;
    const uint32_t r = ((c & 0xffu) * W + s.z + h) / n;
    const uint32_t g = (((c >> 8) & 0xffu) * W + s.y + h) / n;
    const uint32_t b = (((c >> 16) & 0xffu) * W + s.x + h) / n;
    return r | (g << 8) | (b << 16) | (min(n, (uint32_t)wcap) << 24);
}

struct CameraParams {
    Aff d2c;                         // depth camera frame -> colour camera frame
    float fx, fy, cx, cy;            // colour intrinsics
    float fcols, frows;              // colour image size
    int cell;                        // colour pixels per map cell and axis
};

// a df_color_camera with its map's cell (df_color_map_dims) as the kernels take it
inline CameraParams camera_params(const df_color_camera &cam, int cell)
{
    CameraParams c;
    c.d2c = make_aff(cam.depth_to_color);
    c.fx = cam.intr.fx; c.fy = cam.intr.fy; c.cx = cam.intr.cx; c.cy = cam.intr.cy;
    c.fcols = (float)cam.cols; c.frows = (float)cam.rows;
    c.cell = cell;
    return c;
}

// the depth pixel's point in the colour camera and its colour pixel (u, v): false when it does not land in the colour image.  LENS: through
// the colour camera's lens (lens.cuh); the instances without it ignore `lens` and are the pinhole projection
template <bool LENS>
__device__ __forceinline__ bool to_color(const CameraParams &c, const df_lens &lens, const float3 pd, float3 &pc, float &u, float &v)
{
    pc = aff_mul(c.d2c, pd);
    if constexpr (LENS) {
        float xd, yd;
        if (!lens_distort(lens, pc.x / pc.z, pc.y / pc.z, xd, yd)) return false;
        u = __fmaf_rn(c.fx, xd, c.cx);
        v = __fmaf_rn(c.fy, yd, c.cy);
    } else {
        u = __fmaf_rn(c.fx, pc.x / pc.z, c.cx);
        v = __fmaf_rn(c.fy, pc.y / pc.z, c.cy);
    }
    return pc.z > 0 && u >= 0 && v >= 0 && u < c.fcols && v < c.frows;   // a NaN fails every comparison
}

struct OcclusionParams {
    CameraParams cam;
    const uint32_t *map; size_t mpitch;
    float tol;                       // DF_COLOR_OCCLUSION * trunc_dist
};

// the colour camera's pixel of the depth-frame point vc: its colour projection and the occlusion test, then the pixel of bgra; false where
// the camera does not see vc (df_integrate_color_camera's voxels, df_frame_intensity's level-0 points,
// df_integrate_warped_color's warped voxels)
template <bool LENS>
__device__ __forceinline__ bool camera_sample(const OcclusionParams &o, const df_lens &lens, const uchar4 *bgra, size_t cpitch, float3 vc, uchar4 &smp)
{
    float3 pc;
    float u, v;
    if (!to_color<LENS>(o.cam, lens, vc, pc, u, v)) return false;
    const int iu = (int)u, iv = (int)v;
    const uint32_t zmin = __ldg(row_ptr(o.map, o.mpitch, iv / o.cam.cell) + iu / o.cam.cell);
    if (zmin == 0xffffffffu) return false;                         // no depth pixel lands in this cell
    if (pc.z > __uint_as_float(zmin) + o.tol) return false;        // the colour camera sees something nearer here
    smp = __ldg(row_ptr(bgra, cpitch, iv) + iu);
    return true;
}

}  // namespace dfb
