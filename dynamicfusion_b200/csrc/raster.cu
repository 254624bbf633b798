// raster.cu -- deterministic z-buffer rasteriser of a triangle mesh into the ray-cast's point / normal maps and a per-pixel triangle index
// (df_raster_mesh; the rule is written out once in include/dfusion.h).  Used to render the canonical and the live (warped) mesh of the frame
// loop from any camera (df_kinfu_render).  tests/raster_oracle.c implements the same rule operation for operation; the two agree bit for bit.
//
// Passes (5 launches, one stream):
//   clear     z-buffer keys to ~0, the large-triangle queue counter and the stats to 0
//   vertex    one thread per vertex: camera frame point (float4) and 24.8 fixed-point image position (int2; x = INT_MIN: skipped vertex)
//   triangle  one thread per triangle: bad index / skipped vertex -> stats[1], back-facing or zero area -> stats[0]; a clipped bounding box
//             of at most RASTER_SMALL x RASTER_SMALL pixel samples is drawn here (stats[2]), a larger one goes to the queue (stats[3])
//   large     one warp per queued triangle, the lanes stride over its bounding box
//   resolve   one thread per pixel: the winning key's triangle, its depth recomputed by the same function, written as point / normal / index
// Drawing a covered sample is one 64-bit atomicMin of (float bits of t) << 32 | triangle index: the nearest surface wins, a tie goes to the
// smaller index, and the result depends neither on the launch order nor on the queue's order.
#include "df_common.cuh"
#include <climits>

using namespace dfb;

namespace {

constexpr int RASTER_SUB_BITS = 8;                 // sub-pixel bits of the fixed-point image coordinates
constexpr float RASTER_GUARD = 16777216.f;         // 2^16 pixels in fixed point (2^24): edge functions stay below 2^51 in int64
constexpr int RASTER_SMALL = 8;                    // bounding boxes up to 8 x 8 samples are drawn by the triangle pass itself
constexpr int RASTER_LARGE_WARPS = 8;              // warps per block of the large-triangle pass

struct RasterWs {
    unsigned long long *zbuf;                      // cols * rows keys
    float4 *cam;                                   // n_verts camera-frame points
    int2 *fix;                                     // n_verts fixed-point positions
    int *queue;                                    // n_tris triangle indices
    int *qcount;                                   // 1
};

size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

RasterWs raster_ws(void *ws, int n_verts, int n_tris, int cols, int rows)
{
    char *b = (char *)ws;
    RasterWs w;
    w.zbuf = (unsigned long long *)b; b += align256((size_t)cols * rows * 8);
    w.cam = (float4 *)b;              b += align256((size_t)n_verts * 16);
    w.fix = (int2 *)b;                b += align256((size_t)n_verts * 8);
    w.queue = (int *)b;               b += align256((size_t)n_tris * 4);
    w.qcount = (int *)b;
    return w;
}

struct RasterCam { float fx, fy, cx, cy, finvx, finvy; int cols, rows; };

// dot and cross of the rule: plain IEEE products and sums, left to right (the unit is compiled with -fmad=false)
__device__ __forceinline__ float rdot(const float3 a, const float3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
__device__ __forceinline__ float3 rcross(const float3 a, const float3 b)
{ return make_float3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x); }

// the pixel's ray, Reprojector(x, y, 1.f) as the ray-cast builds it
__device__ __forceinline__ float3 pixel_ray(const RasterCam &c, int i, int j)
{ return make_float3(((float)i - c.cx) * c.finvx, ((float)j - c.cy) * c.finvy, 1.f); }

struct Tri {
    long long ax[3], ay[3], dx[3], dy[3];          // edge k runs from vertex k to vertex k+1 of the positively wound (swapped) triangle
    int bias[3];                                   // 0 on a top or left edge (a sample on it is covered), 1 otherwise
    int x0, x1, y0, y1;                            // clipped bounding box of the pixel samples, inclusive
    float3 n; float num;                           // face normal cross(c1 - c0, c2 - c0) in the mesh's order, and dot(n, c0)
};

// 0: draw, 1: back-facing or zero area (stats[0]), 2: skipped (stats[1])
__device__ __forceinline__ int tri_setup(const int32_t *tris, int t, int n_verts, const float4 *cam, const int2 *fix, const RasterCam &c, Tri &T)
{
    const int i0 = tris[3 * (size_t)t], i1 = tris[3 * (size_t)t + 1], i2 = tris[3 * (size_t)t + 2];
    if ((unsigned)i0 >= (unsigned)n_verts || (unsigned)i1 >= (unsigned)n_verts || (unsigned)i2 >= (unsigned)n_verts) return 2;
    const int2 f0 = fix[i0], f1 = fix[i1], f2 = fix[i2];
    if (f0.x == INT_MIN || f1.x == INT_MIN || f2.x == INT_MIN) return 2;
    const long long area = (long long)(f1.x - f0.x) * (f2.y - f0.y) - (long long)(f1.y - f0.y) * (f2.x - f0.x);
    if (area >= 0) return 1;                       // camera-facing triangles have a negative area (image v points down)
    const int2 v[3] = {f0, f2, f1};                // swapped: positive area, inside = every edge function > 0
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const int2 a = v[k], b = v[k == 2 ? 0 : k + 1];
        T.ax[k] = a.x; T.ay[k] = a.y;
        T.dx[k] = (long long)b.x - a.x; T.dy[k] = (long long)b.y - a.y;
        T.bias[k] = (T.dy[k] < 0 || (T.dy[k] == 0 && T.dx[k] > 0)) ? 0 : 1;
    }
    const int mnx = min(f0.x, min(f1.x, f2.x)), mxx = max(f0.x, max(f1.x, f2.x));
    const int mny = min(f0.y, min(f1.y, f2.y)), mxy = max(f0.y, max(f1.y, f2.y));
    T.x0 = max((mnx + 255) >> RASTER_SUB_BITS, 0); T.x1 = min(mxx >> RASTER_SUB_BITS, c.cols - 1);
    T.y0 = max((mny + 255) >> RASTER_SUB_BITS, 0); T.y1 = min(mxy >> RASTER_SUB_BITS, c.rows - 1);
    const float4 q0 = cam[i0], q1 = cam[i1], q2 = cam[i2];
    const float3 c0 = make_float3(q0.x, q0.y, q0.z);
    T.n = rcross(make_float3(q1.x - q0.x, q1.y - q0.y, q1.z - q0.z), make_float3(q2.x - q0.x, q2.y - q0.y, q2.z - q0.z));
    T.num = rdot(T.n, c0);
    return 0;
}

__device__ __forceinline__ bool covers(const Tri &T, int i, int j)
{
    const long long px = (long long)i << RASTER_SUB_BITS, py = (long long)j << RASTER_SUB_BITS;
    bool in = true;
#pragma unroll
    for (int k = 0; k < 3; ++k) in = in && T.dx[k] * (py - T.ay[k]) - T.dy[k] * (px - T.ax[k]) >= T.bias[k];
    return in;
}

__device__ __forceinline__ void draw_sample(const Tri &T, int t, int i, int j, const RasterCam &c, unsigned long long *zbuf)
{
    if (!covers(T, i, j)) return;
    const float tz = T.num / rdot(T.n, pixel_ray(c, i, j));
    if (!(tz > 0.f && tz < INFINITY)) return;
    const unsigned long long key = ((unsigned long long)__float_as_uint(tz) << 32) | (unsigned)t;
    unsigned long long *z = zbuf + (size_t)j * c.cols + i;
    if (key < __ldcg(z)) atomicMin(z, key);        // a stale read is never below the true minimum: skipping is exact
}

__device__ __forceinline__ void warp_count(unsigned long long *stats, int slot, bool pred)
{
    const unsigned m = __ballot_sync(0xffffffffu, pred);
    if (stats && (threadIdx.x & 31) == 0 && m) atomicAdd(stats + slot, (unsigned long long)__popc(m));
}

__global__ void __launch_bounds__(256) raster_clear_kernel(unsigned long long *zbuf, int n, int *qcount, unsigned long long *stats)
{
    DF_PDL_ENTRY();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) zbuf[i] = ~0ull;
    if (i == 0) *qcount = 0;
    if (stats && i < 5) stats[i] = 0;
}

__global__ void __launch_bounds__(256) raster_vertex_kernel(const float *verts, int n, int vstride, Aff w2c, RasterCam c, float4 *cam, int2 *fix)
{
    DF_PDL_ENTRY();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float *v = verts + (size_t)i * vstride;
    const float x = v[0], y = v[1], z = v[2];
    // cv::Affine3f * Vec3f, m0*x + m1*y + m2*z + m3 left to right, as to_canonical_kernel evaluates it
    const float cx = w2c.r0.x * x + w2c.r0.y * y + w2c.r0.z * z + w2c.t.x;
    const float cy = w2c.r1.x * x + w2c.r1.y * y + w2c.r1.z * z + w2c.t.y;
    const float cz = w2c.r2.x * x + w2c.r2.y * y + w2c.r2.z * z + w2c.t.z;
    cam[i] = make_float4(cx, cy, cz, 0.f);
    int2 f = make_int2(INT_MIN, INT_MIN);
    if (isfinite(cx) && isfinite(cy) && isfinite(cz) && cz >= DF_RASTER_NEAR) {
        const float su = __fmaf_rn(c.fx, cx / cz, c.cx) * 256.f, sv = __fmaf_rn(c.fy, cy / cz, c.cy) * 256.f;   // exact scaling by 2^8
        if (fabsf(su) <= RASTER_GUARD && fabsf(sv) <= RASTER_GUARD) f = make_int2(__float2int_rn(su), __float2int_rn(sv));
    }
    fix[i] = f;
}

__global__ void __launch_bounds__(256) raster_triangle_kernel(const int32_t *tris, int n_tris, int n_verts, const float4 *cam, const int2 *fix,
                                                              RasterCam c, unsigned long long *zbuf, int *queue, int *qcount,
                                                              unsigned long long *stats)
{
    DF_PDL_ENTRY();
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    Tri T;
    const int st = t < n_tris ? tri_setup(tris, t, n_verts, cam, fix, c, T) : -1;
    const bool draw = st == 0;
    const bool small = draw && T.x1 - T.x0 < RASTER_SMALL && T.y1 - T.y0 < RASTER_SMALL;
    const bool large = draw && !small;
    warp_count(stats, 0, st == 1);
    warp_count(stats, 1, st == 2);
    warp_count(stats, 2, small);
    warp_count(stats, 3, large);
    // warp-aggregated append to the large-triangle queue
    const unsigned m = __ballot_sync(0xffffffffu, large);
    if (m) {
        const int lane = threadIdx.x & 31, leader = __ffs(m) - 1;
        int base = 0;
        if (lane == leader) base = atomicAdd(qcount, __popc(m));
        base = __shfl_sync(0xffffffffu, base, leader);
        if (large) queue[base + __popc(m & ((1u << lane) - 1))] = t;
    }
    if (!small) return;
    for (int j = T.y0; j <= T.y1; ++j)
        for (int i = T.x0; i <= T.x1; ++i) draw_sample(T, t, i, j, c, zbuf);
}

__global__ void __launch_bounds__(32 * RASTER_LARGE_WARPS) raster_large_kernel(const int32_t *tris, int n_verts, const float4 *cam, const int2 *fix,
                                                                              RasterCam c, unsigned long long *zbuf, const int *queue,
                                                                              const int *qcount)
{
    DF_PDL_ENTRY();
    const int lane = threadIdx.x & 31;
    const int nq = *qcount;
    for (int q = blockIdx.x * RASTER_LARGE_WARPS + (threadIdx.x >> 5); q < nq; q += gridDim.x * RASTER_LARGE_WARPS) {
        const int t = queue[q];
        Tri T;
        tri_setup(tris, t, n_verts, cam, fix, c, T);  // queued triangles are drawn: the status is 0
        const int w = T.x1 - T.x0 + 1, n = w * (T.y1 - T.y0 + 1);
        for (int p = lane; p < n; p += 32) {
            const int j = p / w;
            draw_sample(T, t, T.x0 + p - j * w, T.y0 + j, c, zbuf);
        }
    }
}

__global__ void __launch_bounds__(256) raster_resolve_kernel(const unsigned long long *zbuf, const int32_t *tris, const float4 *cam, RasterCam c,
                                                             int32_t *tri_ids, size_t tpitch, float4 *points, size_t ppitch, float4 *normals,
                                                             size_t npitch, unsigned long long *stats)
{
    DF_PDL_ENTRY();
    const int i = blockIdx.x * blockDim.x + threadIdx.x, j = blockIdx.y * blockDim.y + threadIdx.y;
    const bool in = i < c.cols && j < c.rows;
    const unsigned long long key = in ? zbuf[(size_t)j * c.cols + i] : ~0ull;
    const bool hit = key != ~0ull;
    warp_count(stats, 4, hit);
    if (!in) return;
    const float nanv = qnan();
    float4 P = make_float4(nanv, nanv, nanv, nanv), N = P;
    int id = -1;
    if (hit) {
        id = (int)(unsigned)key;
        const int i0 = tris[3 * (size_t)id], i1 = tris[3 * (size_t)id + 1], i2 = tris[3 * (size_t)id + 2];
        const float4 q0 = cam[i0], q1 = cam[i1], q2 = cam[i2];
        const float3 n = rcross(make_float3(q1.x - q0.x, q1.y - q0.y, q1.z - q0.z), make_float3(q2.x - q0.x, q2.y - q0.y, q2.z - q0.z));
        const float3 d = pixel_ray(c, i, j);
        const float t = rdot(n, make_float3(q0.x, q0.y, q0.z)) / rdot(n, d);   // the function draw_sample evaluated
        const float len = sqrtf(rdot(n, n));
        P = make_float4(d.x * t, d.y * t, t, 0.f);
        N = make_float4(n.x / len, n.y / len, n.z / len, 0.f);
    }
    row_ptr(points, ppitch, j)[i] = P;
    row_ptr(normals, npitch, j)[i] = N;
    if (tri_ids) row_ptr(tri_ids, tpitch, j)[i] = id;
}

// df_mesh_correspond: one thread per pixel; the drawn triangle's corners are recomputed exactly as raster_vertex_kernel computes them
__global__ void __launch_bounds__(256) correspond_kernel(const int32_t *tri_ids, size_t tpitch, const float4 *points, size_t ppitch,
                                                         const float *verts, const float *src, int n_verts, int vstride, const int32_t *tris,
                                                         int n_tris, Aff w2c, int cols, int rows, const float4 *target, size_t gpitch,
                                                         float max_dist, float4 *out_pts, size_t opitch, float4 *out_nrm, size_t npitch)
{
    DF_PDL_ENTRY();
    const int i = blockIdx.x * blockDim.x + threadIdx.x, j = blockIdx.y * blockDim.y + threadIdx.y;
    if (i >= cols || j >= rows) return;
    const float nanv = qnan();
    float4 S = make_float4(nanv, nanv, nanv, nanv), N = S;
    const int id = row_ptr(tri_ids, tpitch, j)[i];
    if (id >= 0 && id < n_tris) {
        const int ix[3] = {tris[3 * (size_t)id], tris[3 * (size_t)id + 1], tris[3 * (size_t)id + 2]};
        bool ok = (unsigned)ix[0] < (unsigned)n_verts && (unsigned)ix[1] < (unsigned)n_verts && (unsigned)ix[2] < (unsigned)n_verts;
        const float4 P4 = row_ptr(points, ppitch, j)[i];
        const float3 P = make_float3(P4.x, P4.y, P4.z);
        if (ok && target) {
            const float4 T = row_ptr(target, gpitch, j)[i];
            const float dx = T.x - P.x, dy = T.y - P.y, dz = T.z - P.z;
            ok = !isnan(T.x) && !isnan(T.y) && !isnan(T.z) && !(dx * dx + dy * dy + dz * dz > max_dist * max_dist);
        }
        if (ok) {
            float3 c[3], s[3];
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                const float *v = verts + (size_t)ix[k] * vstride, *w = src + (size_t)ix[k] * vstride;
                const float x = v[0], y = v[1], z = v[2];
                c[k] = make_float3(w2c.r0.x * x + w2c.r0.y * y + w2c.r0.z * z + w2c.t.x, w2c.r1.x * x + w2c.r1.y * y + w2c.r1.z * z + w2c.t.y,
                                   w2c.r2.x * x + w2c.r2.y * y + w2c.r2.z * z + w2c.t.z);
                s[k] = make_float3(w[0], w[1], w[2]);
            }
            const float3 e0 = make_float3(c[1].x - c[0].x, c[1].y - c[0].y, c[1].z - c[0].z);
            const float3 e1 = make_float3(c[2].x - c[0].x, c[2].y - c[0].y, c[2].z - c[0].z);
            const float3 q = make_float3(P.x - c[0].x, P.y - c[0].y, P.z - c[0].z);
            const float d00 = rdot(e0, e0), d01 = rdot(e0, e1), d11 = rdot(e1, e1), d20 = rdot(q, e0), d21 = rdot(q, e1);
            const float den = d00 * d11 - d01 * d01;
            if (isfinite(den) && den != 0.f) {
                const float b1 = (d11 * d20 - d01 * d21) / den, b2 = (d00 * d21 - d01 * d20) / den, b0 = 1.f - b1 - b2;
                S = make_float4((b0 * s[0].x + b1 * s[1].x) + b2 * s[2].x, (b0 * s[0].y + b1 * s[1].y) + b2 * s[2].y,
                                (b0 * s[0].z + b1 * s[1].z) + b2 * s[2].z, 0.f);
                const float3 n = rcross(make_float3(s[1].x - s[0].x, s[1].y - s[0].y, s[1].z - s[0].z),
                                        make_float3(s[2].x - s[0].x, s[2].y - s[0].y, s[2].z - s[0].z));
                const float len = sqrtf(rdot(n, n));
                N = make_float4(n.x / len, n.y / len, n.z / len, 0.f);
            }
        }
    }
    row_ptr(out_pts, opitch, j)[i] = S;
    row_ptr(out_nrm, npitch, j)[i] = N;
}

}  // namespace

extern "C" int df_mesh_correspond(const int32_t *tri_ids, size_t tri_pitch, const float *points, size_t points_pitch, const float *verts,
                                  const float *src_verts, int n_verts, int vstride, const int32_t *tris, int n_tris, df_aff3f world2cam, int cols,
                                  int rows, const float *target, size_t target_pitch, float max_dist, float *src_points, size_t src_points_pitch,
                                  float *src_normals, size_t src_normals_pitch, void *stream)
{
    if (n_verts < 0 || n_tris < 0 || (vstride != 3 && vstride != 4) || cols <= 0 || rows <= 0 || cols > DF_RASTER_MAX_DIM ||
        rows > DF_RASTER_MAX_DIM || !tri_ids || !points || !src_points || !src_normals || (n_verts > 0 && (!verts || !src_verts)) ||
        (n_tris > 0 && !tris) || tri_pitch < (size_t)cols * 4 || tri_pitch % 4 || points_pitch < (size_t)cols * 16 || points_pitch % 16 ||
        src_points_pitch < (size_t)cols * 16 || src_points_pitch % 16 || src_normals_pitch < (size_t)cols * 16 || src_normals_pitch % 16 ||
        (target && (target_pitch < (size_t)cols * 16 || target_pitch % 16)))
        return (int)cudaErrorInvalidValue;
    launch_pdl(correspond_kernel, dim3(div_up(cols, 32), div_up(rows, 8)), dim3(32, 8), 0, (cudaStream_t)stream, tri_ids, tri_pitch,
               (const float4 *)points, points_pitch, verts, src_verts, n_verts, vstride, tris, n_tris, make_aff(world2cam), cols, rows,
               (const float4 *)target, target_pitch, max_dist, (float4 *)src_points, src_points_pitch, (float4 *)src_normals, src_normals_pitch);
    DF_LAUNCH_CHECK();
    return 0;
}

extern "C" size_t df_raster_workspace_bytes(int n_verts, int n_tris, int cols, int rows)
{
    if (n_verts < 0 || n_tris < 0 || cols <= 0 || rows <= 0) return 0;
    return align256((size_t)cols * rows * 8) + align256((size_t)n_verts * 16) + align256((size_t)n_verts * 8) + align256((size_t)n_tris * 4) + 256;
}

extern "C" int df_raster_mesh(const float *verts, int n_verts, int vstride, const int32_t *tris, int n_tris, df_aff3f world2cam, df_intr intr,
                              int cols, int rows, int32_t *tri_ids, size_t tri_pitch, float *points, size_t points_pitch, float *normals,
                              size_t normals_pitch, unsigned long long *stats_dev, void *workspace, void *stream)
{
    if (n_verts < 0 || n_tris < 0 || (vstride != 3 && vstride != 4) || cols <= 0 || rows <= 0 || cols > DF_RASTER_MAX_DIM ||
        rows > DF_RASTER_MAX_DIM || !points || !normals || !workspace || (n_verts > 0 && !verts) || (n_tris > 0 && !tris) ||
        points_pitch < (size_t)cols * 16 || normals_pitch < (size_t)cols * 16 || points_pitch % 16 || normals_pitch % 16 ||
        (tri_ids && (tri_pitch < (size_t)cols * 4 || tri_pitch % 4)))
        return (int)cudaErrorInvalidValue;
    const cudaStream_t s = (cudaStream_t)stream;
    const RasterWs w = raster_ws(workspace, n_verts, n_tris, cols, rows);
    RasterCam c;
    c.fx = intr.fx; c.fy = intr.fy; c.cx = intr.cx; c.cy = intr.cy;
    c.finvx = 1.f / intr.fx; c.finvy = 1.f / intr.fy;                 // Reprojector ctor, as the ray-cast computes it
    c.cols = cols; c.rows = rows;
    const int npix = cols * rows;
    launch_pdl(raster_clear_kernel, dim3(div_up(npix, 256)), dim3(256), 0, s, w.zbuf, npix, w.qcount, stats_dev);
    if (n_verts > 0)
        launch_pdl(raster_vertex_kernel, dim3(div_up(n_verts, 256)), dim3(256), 0, s, verts, n_verts, vstride, make_aff(world2cam), c, w.cam, w.fix);
    if (n_tris > 0) {
        launch_pdl(raster_triangle_kernel, dim3(div_up(n_tris, 256)), dim3(256), 0, s, (const int32_t *)tris, n_tris, n_verts,
                   (const float4 *)w.cam, (const int2 *)w.fix, c, w.zbuf, w.queue, w.qcount, stats_dev);
        const int grid = min(div_up(n_tris, RASTER_LARGE_WARPS), 16 * DF_NUM_SMS);
        launch_pdl(raster_large_kernel, dim3(grid), dim3(32 * RASTER_LARGE_WARPS), 0, s, (const int32_t *)tris, n_verts, (const float4 *)w.cam,
                   (const int2 *)w.fix, c, w.zbuf, (const int *)w.queue, (const int *)w.qcount);
    }
    launch_pdl(raster_resolve_kernel, dim3(div_up(cols, 32), div_up(rows, 8)), dim3(32, 8), 0, s, (const unsigned long long *)w.zbuf,
               (const int32_t *)tris, (const float4 *)w.cam, c, tri_ids, tri_pitch, (float4 *)points, points_pitch, (float4 *)normals,
               normals_pitch, stats_dev);
    DF_LAUNCH_CHECK();
    return 0;
}
