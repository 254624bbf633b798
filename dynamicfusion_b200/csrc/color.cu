// color.cu -- the optional colour volume: fusing a BGRA frame into it, registered to the depth or from a colour camera with its own
// calibration, and sampling it at points (sm_90a).
//
// The rules are written out in include/dfusion.h (df_integrate_color, df_sample_colors, df_color_depth_map, df_integrate_color_camera) and
// restated in plain C by tests/color_oracle.c and tests/color_camera_oracle.c (through a lens: tests/lens_oracle.c); the kernels below follow them operation for operation.  The colour volume never feeds back into the TSDF volume or the warp field, and into the poses only under
// DF_KINFU_COLOR_TRACKING: there df_frame_intensity and df_model_intensity (rules in include/dfusion.h, restated by tests/color_track_oracle.c) give
// the intensity maps of the photometric ICP rows (csrc/icp.cu, df_icp_accumulate_color).
#include "volscan.cuh"
#include "color_sample.cuh"
#include "lens.cuh"
#include "../../include/df_hostmath.h"
#include <algorithm>
#include <cmath>
#include <cstring>

using namespace dfb;

namespace {

struct ColorParams {
    uint32_t *colors;
    float vsx, vsy, vsz;
    float band;                      // DF_COLOR_BAND * trunc_dist
    int wcap;                        // min(max_weight, 255)
    const unsigned short *dists; size_t dpitch;
    const uchar4 *bgra; size_t cpitch;
    float fcols, frows;
    Aff vol2cam;
    float fx, fy, cx, cy;
};

// the depth side of both integrate rules, then sample(vc, u, v, s): the voxel's camera-frame position and depth pixel (u, v) give its colour
// sample s, or false to skip it; false also when a depth-side test skips the voxel
template <class Sample>
__device__ __forceinline__ bool depth_gate(const ColorParams &p, int x, int y, int z, uchar4 &s, Sample sample)
{
    const float3 vc = aff_mul(p.vol2cam, make_float3((float)x * p.vsx, (float)y * p.vsy, (float)z * p.vsz));
    const float u = __fmaf_rn(p.fx, vc.x / vc.z, p.cx);
    const float v = __fmaf_rn(p.fy, vc.y / vc.z, p.cy);
    if (u < 0 || v < 0 || u >= p.fcols || v >= p.frows) return false;
    if (vc.z <= 0) return false;
    if (!(u == u) || !(v == v)) return false;
    const float Dp = half_bits_to_float(__ldg(row_ptr(p.dists, p.dpitch, (int)v) + (int)u));
    if (Dp == 0) return false;
    const float sdf = Dp - sqrtf(dot3(vc, vc));
    if (!(fabsf(sdf) <= p.band)) return false;
    return sample(vc, u, v, s);
}

// the frame's colour sample for voxel (x, y, z), registered image: false when the rule skips the voxel
__device__ __forceinline__ bool color_gate(const ColorParams &p, int x, int y, int z, uchar4 &s)
{
    return depth_gate(p, x, y, z, s, [&](float3, float u, float v, uchar4 &smp) {
        smp = __ldg(row_ptr(p.bgra, p.cpitch, (int)v) + (int)u);
        return true;
    });
}

// the walk both integrate kernels share: gate(x, y, z, s) gives voxel (x, y, z)'s sample or skips it; one read-modify-write per changed quad
template <int VX, class Gate> __device__ __forceinline__ void color_walk(const VolumeWalk &w, const ColorParams &p, Gate gate)
{
#pragma unroll
    for (int i = 0; i < WALK_QPT; ++i) {
        const size_t v0 = quad_voxel<VX>(i);
        if (quad_skipped(w, v0)) continue;
        const QuadCoord c = quad_coord(w, v0);
        uchar4 s[VX];
        unsigned mask = 0;
#pragma unroll
        for (int j = 0; j < VX; ++j)
            if (gate(c.x0 + j, c.y, c.z, s[j])) mask |= 1u << j;
        if (!mask) continue;
        if (VX == 4) {
            uint4 *q = reinterpret_cast<uint4 *>(p.colors + v0);
            const uint4 old = *q;
            uint4 val = old;
            if (mask & 1u) val.x = color_update(val.x, s[0], p.wcap);
            if (mask & 2u) val.y = color_update(val.y, s[1 % VX], p.wcap);
            if (mask & 4u) val.z = color_update(val.z, s[2 % VX], p.wcap);
            if (mask & 8u) val.w = color_update(val.w, s[3 % VX], p.wcap);
            if (val.x != old.x || val.y != old.y || val.z != old.z || val.w != old.w) *q = val;
        } else {
            const uint32_t old = p.colors[v0], val = color_update(old, s[0], p.wcap);
            if (val != old) p.colors[v0] = val;
        }
    }
}

template <int VX>
__global__ void __launch_bounds__(WALK_THREADS) integrate_color_kernel(const VolumeWalk w, const ColorParams p)
{
    DF_PDL_ENTRY();
    color_walk<VX>(w, p, [&](int x, int y, int z, uchar4 &s) { return color_gate(p, x, y, z, s); });
}

// ---- a colour camera with its own calibration (df_color_depth_map, df_integrate_color_camera) -------------------------------------

template <bool LENS>
__global__ void __launch_bounds__(256) color_depth_map_kernel(const unsigned short *depth, size_t dpitch, int cols, int rows, float finvx, float finvy,
                                                              float dcx, float dcy, const CameraParams c, uint32_t *map, size_t mpitch,
                                                              const df_lens lens)
{
    DF_PDL_ENTRY();
    const int i = blockIdx.x * blockDim.x + threadIdx.x, j = blockIdx.y * blockDim.y + threadIdx.y;
    if (i >= cols || j >= rows) return;
    const unsigned short d = row_ptr(depth, dpitch, j)[i];
    if (d == 0) return;
    const float z = (float)d * 0.001f;
    const float3 pd = make_float3(z * ((float)i - dcx) * finvx, z * ((float)j - dcy) * finvy, z);   // df_points_normals' reprojection
    float3 pc;
    float u, v;
    if (!to_color<LENS>(c, lens, pd, pc, u, v)) return;
    atomicMin(row_ptr(map, mpitch, (int)v / c.cell) + (int)u / c.cell, __float_as_uint(pc.z));   // positive floats order as their bits
}

// the colour camera's sample for voxel (x, y, z): the depth-side gate, then the colour projection and the occlusion test
template <bool LENS>
__device__ __forceinline__ bool camera_gate(const ColorParams &p, const OcclusionParams &o, const df_lens &lens, int x, int y, int z, uchar4 &s)
{
    return depth_gate(p, x, y, z, s, [&](float3 vc, float, float, uchar4 &smp) { return camera_sample<LENS>(o, lens, p.bgra, p.cpitch, vc, smp); });
}

template <int VX, bool LENS>
__global__ void __launch_bounds__(WALK_THREADS) integrate_color_camera_kernel(const VolumeWalk w, const ColorParams p, const OcclusionParams o,
                                                                              const df_lens lens)
{
    DF_PDL_ENTRY();
    color_walk<VX>(w, p, [&](int x, int y, int z, uchar4 &s) { return camera_gate<LENS>(p, o, lens, x, y, z, s); });
}

__global__ void __launch_bounds__(256) sample_colors_kernel(const SampleParams p)
{
    DF_PDL_ENTRY();
    const int i = blockIdx.x * blockDim.x + threadIdx.x, j = blockIdx.y;
    int n = p.cols;
    if (p.count) n = min(n, *p.count);
    if (i >= n) return;
    const float *pt = (const float *)(p.points + (size_t)j * p.ppitch + (size_t)i * p.stride * 4);
    *(uint32_t *)(p.rgba + (size_t)j * p.opitch + (size_t)i * 4) = sample_color(p, pt[0], pt[1], pt[2]);
}

// ---- colour tracking: the intensity maps of the frame and of the model (df_frame_intensity, df_model_intensity) -------------------------

__device__ __forceinline__ float luma(uint32_t r, uint32_t g, uint32_t b) { return (float)((77u * r + 150u * g + 29u * b + 128u) >> 8) / 255.f; }

struct FrameIntensityParams {
    const uchar4 *bgra; size_t cpitch;
    int cols, rows;
    bool cam;                        // through the colour camera (o, points) or the registered image
    OcclusionParams o;
    const float4 *points; size_t ppitch;
    float *out; size_t opitch;
};

template <bool LENS> __global__ void __launch_bounds__(256) frame_intensity_kernel(const FrameIntensityParams p, const df_lens lens)
{
    DF_PDL_ENTRY();
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= p.cols || y >= p.rows) return;
    float I = qnan();
    uchar4 c;
    if (!p.cam) {
        c = __ldg(row_ptr(p.bgra, p.cpitch, y) + x);
        I = luma(c.z, c.y, c.x);
    } else {
        const float4 pt = __ldg(row_ptr(p.points, p.ppitch, y) + x);
        if (!isnan(pt.x) && camera_sample<LENS>(p.o, lens, p.bgra, p.cpitch, make_float3(pt.x, pt.y, pt.z), c)) I = luma(c.z, c.y, c.x);
    }
    row_ptr(p.out, p.opitch, y)[x] = I;
}

// level l from level l - 1 (cols x rows: level l's size): the mean of the valid values of each 2 x 2 block
__global__ void __launch_bounds__(256) intensity_down_kernel(const float *src, size_t spitch, float *dst, size_t dpitch, int cols, int rows)
{
    DF_PDL_ENTRY();
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= cols || y >= rows) return;
    float s = 0.f;
    int n = 0;
#pragma unroll
    for (int dy = 0; dy < 2; ++dy)
#pragma unroll
        for (int dx = 0; dx < 2; ++dx) {
            const float v = __ldg(row_ptr(src, spitch, 2 * y + dy) + 2 * x + dx);
            if (!isnan(v)) { s = s + v; ++n; }
        }
    row_ptr(dst, dpitch, y)[x] = n ? s / (float)n : qnan();
}

constexpr int MI_LEVELS = 4, MI_BX = 32, MI_BY = 8;
struct ModelIntensityParams {
    SampleParams s;                  // colors, dims, voxel size, offset 0 and world2vol = cam2vol
    int cols[MI_LEVELS], rows[MI_LEVELS];
    const float4 *points[MI_LEVELS]; size_t ppitch[MI_LEVELS];
    float4 *maps[MI_LEVELS]; size_t mpitch[MI_LEVELS];
};

// one 32 x 8 tile of level blockIdx.z: the intensities of the tile and a one-pixel halo are sampled once into shared memory, then every
// pixel takes its central differences from there
__global__ void __launch_bounds__(MI_BX * MI_BY) model_intensity_kernel(const ModelIntensityParams p)
{
    DF_PDL_ENTRY();
    const int l = blockIdx.z, cols = p.cols[l], rows = p.rows[l];
    const int x0 = blockIdx.x * MI_BX, y0 = blockIdx.y * MI_BY;
    if (x0 >= cols || y0 >= rows) return;                            // the grid covers level 0: the whole block lies outside this level
    __shared__ float I[MI_BY + 2][MI_BX + 2];
    const float4 *pts = p.points[l];
    const size_t ppitch = p.ppitch[l];
    for (int i = threadIdx.y * MI_BX + threadIdx.x; i < (MI_BY + 2) * (MI_BX + 2); i += MI_BX * MI_BY) {
        const int hx = i % (MI_BX + 2), hy = i / (MI_BX + 2), x = x0 - 1 + hx, y = y0 - 1 + hy;
        float v = qnan();
        if (x >= 0 && y >= 0 && x < cols && y < rows) {
            const float4 pt = __ldg(row_ptr(pts, ppitch, y) + x);
            const uint32_t c = sample_color(p.s, pt.x, pt.y, pt.z);
            if (c) v = luma(c & 0xffu, (c >> 8) & 0xffu, (c >> 16) & 0xffu);
        }
        I[hy][hx] = v;
    }
    __syncthreads();
    const int tx = threadIdx.x, ty = threadIdx.y, x = x0 + tx, y = y0 + ty;
    if (x >= cols || y >= rows) return;
    const float nan = qnan();
    float4 o = make_float4(nan, nan, nan, nan);
    if (x > 0 && y > 0 && x < cols - 1 && y < rows - 1) {
        const float c = I[ty + 1][tx + 1];
        const float gu = (I[ty + 1][tx + 2] - I[ty + 1][tx]) * 0.5f, gv = (I[ty + 2][tx + 1] - I[ty][tx + 1]) * 0.5f;
        if (!isnan(c) && !isnan(gu) && !isnan(gv)) o = make_float4(c, gu, gv, 0.f);
    }
    row_ptr(p.maps[l], p.mpitch[l], y)[x] = o;
}

}  // namespace

// the depth side shared by both integrate entries (the walk is over the colour array: its 4-voxel / 1-voxel choice follows it)
static ColorParams color_params(const df_volume &vol, uint32_t *colors, const uint16_t *dists, size_t dists_pitch, const void *bgra, size_t bgra_pitch,
                                int cols, int rows, df_aff3f vol2cam, df_intr intr)
{
    ColorParams p;
    p.colors = colors;
    p.vsx = vol.voxel_size[0]; p.vsy = vol.voxel_size[1]; p.vsz = vol.voxel_size[2];
    p.band = DF_COLOR_BAND * vol.trunc_dist;
    p.wcap = vol.max_weight < 255 ? vol.max_weight : 255;
    p.dists = dists; p.dpitch = dists_pitch;
    p.bgra = (const uchar4 *)bgra; p.cpitch = bgra_pitch;
    p.fcols = (float)cols; p.frows = (float)rows;
    p.vol2cam = make_aff(vol2cam);
    p.fx = intr.fx; p.fy = intr.fy; p.cx = intr.cx; p.cy = intr.cy;
    return p;
}

extern "C" int df_integrate_color(df_volume vol, uint32_t *colors, const uint16_t *dists, size_t dists_pitch, const void *bgra,
                                  size_t bgra_pitch, int cols, int rows, df_aff3f vol2cam, df_intr intr, const unsigned char *activity,
                                  void *stream)
{
    if (!colors || !dists || !bgra || cols <= 0 || rows <= 0 || vol.dims[0] <= 0 || vol.dims[1] <= 0 || vol.dims[2] <= 0 ||
        dists_pitch < (size_t)cols * 2 || dists_pitch % 2 || bgra_pitch < (size_t)cols * 4 || bgra_pitch % 4)
        return (int)cudaErrorInvalidValue;
    df_volume cv = vol;
    cv.data = colors;
    const VolumeWalk w = volume_walk(cv, activity);
    const ColorParams p = color_params(vol, colors, dists, dists_pitch, bgra, bgra_pitch, cols, rows, vol2cam, intr);
    if (w.vx == 4) launch_pdl(integrate_color_kernel<4>, dim3(w.nblocks), dim3(WALK_THREADS), 0, (cudaStream_t)stream, w, p);
    else launch_pdl(integrate_color_kernel<1>, dim3(w.nblocks), dim3(WALK_THREADS), 0, (cudaStream_t)stream, w, p);
    DF_LAUNCH_CHECK();
    return 0;
}

static bool finite_all(const float *a, int n)
{
    for (int i = 0; i < n; ++i)
        if (!std::isfinite(a[i])) return false;
    return true;
}

extern "C" int df_color_map_dims(df_intr intr, df_color_camera cam, int *map_cols, int *map_rows, int *cell)
{
    const float ki[4] = {intr.fx, intr.fy, intr.cx, intr.cy}, kc[4] = {cam.intr.fx, cam.intr.fy, cam.intr.cx, cam.intr.cy};
    if (!finite_all(ki, 4) || !(intr.fx > 0) || !(intr.fy > 0) || !finite_all(kc, 4) || !(cam.intr.fx > 0) || !(cam.intr.fy > 0) ||
        !finite_all(cam.depth_to_color.R, 9) || !finite_all(cam.depth_to_color.t, 3) || cam.cols < 1 || cam.cols > 16384 || cam.rows < 1 ||
        cam.rows > 16384)
        return (int)cudaErrorInvalidValue;
    const int c = std::max(1, (int)ceilf(fmaxf(cam.intr.fx / intr.fx, cam.intr.fy / intr.fy)));
    if (cell) *cell = c;
    if (map_cols) *map_cols = (cam.cols + c - 1) / c;
    if (map_rows) *map_rows = (cam.rows + c - 1) / c;
    return 0;
}

// the lens argument of a _lens entry: `use` is false for NULL and for the zero lens (the pinhole instances); an invalid lens is refused
static int lens_arg(const df_lens *lens, bool &use)
{
    use = lens && !lens_is_zero(*lens);
    return lens && df_lens_check(*lens) ? (int)cudaErrorInvalidValue : 0;
}

extern "C" int df_color_depth_map_lens(const uint16_t *depth, size_t depth_pitch, int cols, int rows, df_intr intr, df_color_camera cam,
                                       const df_lens *lens, uint32_t *map, size_t map_pitch, void *stream)
{
    int mcols = 0, mrows = 0, cell = 0;
    bool use_lens = false;
    if (df_color_map_dims(intr, cam, &mcols, &mrows, &cell) || lens_arg(lens, use_lens) || !depth || !map || cols <= 0 || rows <= 0 ||
        depth_pitch < (size_t)cols * 2 || depth_pitch % 2 || map_pitch < (size_t)mcols * 4 || map_pitch % 4)
        return (int)cudaErrorInvalidValue;
    cudaStream_t s = (cudaStream_t)stream;
    if (cudaMemset2DAsync(map, map_pitch, 0xff, (size_t)mcols * 4, mrows, s) != cudaSuccess) return (int)cudaGetLastError();   // every word empty
    const dim3 block(32, 8), grid(div_up(cols, 32), div_up(rows, 8));
    const df_lens L = use_lens ? *lens : df_lens{};
    launch_pdl(use_lens ? color_depth_map_kernel<true> : color_depth_map_kernel<false>, grid, block, 0, s, depth, depth_pitch, cols, rows,
               1.f / intr.fx, 1.f / intr.fy, intr.cx, intr.cy, camera_params(cam, cell), map, map_pitch, L);
    DF_LAUNCH_CHECK();
    return 0;
}

extern "C" int df_color_depth_map(const uint16_t *depth, size_t depth_pitch, int cols, int rows, df_intr intr, df_color_camera cam, uint32_t *map,
                                  size_t map_pitch, void *stream)
{
    return df_color_depth_map_lens(depth, depth_pitch, cols, rows, intr, cam, nullptr, map, map_pitch, stream);
}

extern "C" int df_integrate_color_camera_lens(df_volume vol, uint32_t *colors, const uint16_t *dists, size_t dists_pitch, int cols, int rows,
                                              df_aff3f vol2cam, df_intr intr, df_color_camera cam, const df_lens *lens, const void *bgra,
                                              size_t bgra_pitch, const uint32_t *map, size_t map_pitch, const unsigned char *activity, void *stream)
{
    int mcols = 0, mrows = 0, cell = 0;
    bool use_lens = false;
    if (df_color_map_dims(intr, cam, &mcols, &mrows, &cell) || lens_arg(lens, use_lens) || !colors || !dists || !bgra || !map || cols <= 0 || rows <= 0 || vol.dims[0] <= 0 ||
        vol.dims[1] <= 0 || vol.dims[2] <= 0 || dists_pitch < (size_t)cols * 2 || dists_pitch % 2 || bgra_pitch < (size_t)cam.cols * 4 ||
        bgra_pitch % 4 || map_pitch < (size_t)mcols * 4 || map_pitch % 4)
        return (int)cudaErrorInvalidValue;
    df_volume cv = vol;
    cv.data = colors;
    const VolumeWalk w = volume_walk(cv, activity);
    const ColorParams p = color_params(vol, colors, dists, dists_pitch, bgra, bgra_pitch, cols, rows, vol2cam, intr);
    OcclusionParams o;
    o.cam = camera_params(cam, cell);
    o.map = map; o.mpitch = map_pitch;
    o.tol = DF_COLOR_OCCLUSION * vol.trunc_dist;
    const df_lens L = use_lens ? *lens : df_lens{};
    auto kernel = w.vx == 4 ? (use_lens ? integrate_color_camera_kernel<4, true> : integrate_color_camera_kernel<4, false>)
                            : (use_lens ? integrate_color_camera_kernel<1, true> : integrate_color_camera_kernel<1, false>);
    launch_pdl(kernel, dim3(w.nblocks), dim3(WALK_THREADS), 0, (cudaStream_t)stream, w, p, o, L);
    DF_LAUNCH_CHECK();
    return 0;
}

extern "C" int df_integrate_color_camera(df_volume vol, uint32_t *colors, const uint16_t *dists, size_t dists_pitch, int cols, int rows,
                                         df_aff3f vol2cam, df_intr intr, df_color_camera cam, const void *bgra, size_t bgra_pitch, const uint32_t *map,
                                         size_t map_pitch, const unsigned char *activity, void *stream)
{
    return df_integrate_color_camera_lens(vol, colors, dists, dists_pitch, cols, rows, vol2cam, intr, cam, nullptr, bgra, bgra_pitch, map, map_pitch,
                                          activity, stream);
}

extern "C" int df_sample_colors(df_volume vol, const uint32_t *colors, df_aff3f vol_pose, float offset, const float *points,
                                size_t points_pitch, int stride, int cols, int rows, const int *count_dev, uint32_t *rgba, size_t rgba_pitch,
                                void *stream)
{
    if (!colors || !points || !rgba || cols <= 0 || rows <= 0 || rows > 65535 || (stride != 3 && stride != 4) || vol.dims[0] <= 0 ||
        vol.dims[1] <= 0 || vol.dims[2] <= 0 || points_pitch % 4 || rgba_pitch % 4 ||
        (rows > 1 && (points_pitch < (size_t)cols * stride * 4 || rgba_pitch < (size_t)cols * 4)))
        return (int)cudaErrorInvalidValue;
    float pose12[12], inv12[12];
    memcpy(pose12, vol_pose.R, 36); memcpy(pose12 + 9, vol_pose.t, 12);
    dfh_aff_inv(pose12, inv12);
    df_aff3f inv;
    memcpy(inv.R, inv12, 36); memcpy(inv.t, inv12 + 9, 12);
    SampleParams p;
    p.colors = colors;
    p.Dx = vol.dims[0]; p.Dy = vol.dims[1]; p.Dz = vol.dims[2];
    p.vsx = vol.voxel_size[0]; p.vsy = vol.voxel_size[1]; p.vsz = vol.voxel_size[2]; p.offset = offset;
    p.world2vol = make_aff(inv);
    p.points = (const char *)points; p.ppitch = points_pitch; p.stride = stride;
    p.cols = cols; p.rows = rows;
    p.count = rows == 1 ? count_dev : nullptr;
    p.rgba = (char *)rgba; p.opitch = rgba_pitch;
    launch_pdl(sample_colors_kernel, dim3(div_up(cols, 256), rows), dim3(256), 0, (cudaStream_t)stream, p);
    DF_LAUNCH_CHECK();
    return 0;
}

extern "C" int df_frame_intensity_lens(const void *bgra, size_t bgra_pitch, const df_color_camera *cam, const df_lens *lens, df_intr intr,
                                       const float *points, size_t points_pitch, const uint32_t *map, size_t map_pitch, float trunc_dist, int levels,
                                       const int *cols, const int *rows, float *const *intensity, const size_t *pitch, void *stream)
{
    bool use_lens = false;
    if (lens_arg(lens, use_lens)) return (int)cudaErrorInvalidValue;
    use_lens = use_lens && cam;                                        // the registered image has no colour camera to project through
    if (!bgra || bgra_pitch % 4 || levels < 1 || levels > MI_LEVELS || !cols || !rows || !intensity || !pitch) return (int)cudaErrorInvalidValue;
    for (int l = 0; l < levels; ++l)
        if (!intensity[l] || cols[l] < 1 || rows[l] < 1 || pitch[l] < (size_t)cols[l] * 4 || pitch[l] % 4 ||
            (l > 0 && (cols[l] != cols[l - 1] / 2 || rows[l] != rows[l - 1] / 2)))
            return (int)cudaErrorInvalidValue;
    FrameIntensityParams p = {};
    p.bgra = (const uchar4 *)bgra; p.cpitch = bgra_pitch;
    p.cols = cols[0]; p.rows = rows[0];
    p.out = intensity[0]; p.opitch = pitch[0];
    p.cam = cam != nullptr;
    if (cam) {
        int mcols = 0, mrows = 0, cell = 0;
        if (df_color_map_dims(intr, *cam, &mcols, &mrows, &cell) || !points || points_pitch < (size_t)cols[0] * 16 || points_pitch % 16 || !map ||
            map_pitch < (size_t)mcols * 4 || map_pitch % 4 || bgra_pitch < (size_t)cam->cols * 4)
            return (int)cudaErrorInvalidValue;
        p.o.cam = camera_params(*cam, cell);
        p.o.map = map; p.o.mpitch = map_pitch;
        p.o.tol = DF_COLOR_OCCLUSION * trunc_dist;
        p.points = (const float4 *)points; p.ppitch = points_pitch;
    } else if (bgra_pitch < (size_t)cols[0] * 4)
        return (int)cudaErrorInvalidValue;
    cudaStream_t s = (cudaStream_t)stream;
    const dim3 block(32, 8);
    const df_lens L = use_lens ? *lens : df_lens{};
    launch_pdl(use_lens ? frame_intensity_kernel<true> : frame_intensity_kernel<false>, dim3(div_up(cols[0], 32), div_up(rows[0], 8)), block, 0, s,
               p, L);
    DF_LAUNCH_CHECK();
    for (int l = 1; l < levels; ++l) {
        launch_pdl(intensity_down_kernel, dim3(div_up(cols[l], 32), div_up(rows[l], 8)), block, 0, s, (const float *)intensity[l - 1], pitch[l - 1],
                   intensity[l], pitch[l], cols[l], rows[l]);
        DF_LAUNCH_CHECK();
    }
    return 0;
}

extern "C" int df_frame_intensity(const void *bgra, size_t bgra_pitch, const df_color_camera *cam, df_intr intr, const float *points,
                                  size_t points_pitch, const uint32_t *map, size_t map_pitch, float trunc_dist, int levels, const int *cols,
                                  const int *rows, float *const *intensity, const size_t *pitch, void *stream)
{
    return df_frame_intensity_lens(bgra, bgra_pitch, cam, nullptr, intr, points, points_pitch, map, map_pitch, trunc_dist, levels, cols, rows,
                                   intensity, pitch, stream);
}

extern "C" int df_model_intensity(df_volume vol, const uint32_t *colors, df_aff3f cam2vol, int levels, const int *cols, const int *rows,
                                  const float *const *points, const size_t *points_pitch, float *const *maps, const size_t *maps_pitch, void *stream)
{
    if (!colors || levels < 1 || levels > MI_LEVELS || !cols || !rows || !points || !points_pitch || !maps || !maps_pitch || vol.dims[0] <= 0 ||
        vol.dims[1] <= 0 || vol.dims[2] <= 0)
        return (int)cudaErrorInvalidValue;
    ModelIntensityParams p = {};
    for (int l = 0; l < levels; ++l) {
        if (!points[l] || !maps[l] || cols[l] < 1 || rows[l] < 1 || cols[l] > cols[0] || rows[l] > rows[0] || points_pitch[l] < (size_t)cols[l] * 16 ||
            points_pitch[l] % 16 || maps_pitch[l] < (size_t)cols[l] * 16 || maps_pitch[l] % 16)
            return (int)cudaErrorInvalidValue;
        p.cols[l] = cols[l]; p.rows[l] = rows[l];
        p.points[l] = (const float4 *)points[l]; p.ppitch[l] = points_pitch[l];
        p.maps[l] = (float4 *)maps[l]; p.mpitch[l] = maps_pitch[l];
    }
    p.s.colors = colors;
    p.s.Dx = vol.dims[0]; p.s.Dy = vol.dims[1]; p.s.Dz = vol.dims[2];
    p.s.vsx = vol.voxel_size[0]; p.s.vsy = vol.voxel_size[1]; p.s.vsz = vol.voxel_size[2];
    p.s.offset = 0.f;                                                 // the ray-cast's convention: voxel i at i * vs
    p.s.world2vol = make_aff(cam2vol);
    launch_pdl(model_intensity_kernel, dim3(div_up(cols[0], MI_BX), div_up(rows[0], MI_BY), levels), dim3(MI_BX, MI_BY), 0, (cudaStream_t)stream, p);
    DF_LAUNCH_CHECK();
    return 0;
}
