// extract.cu -- zero-crossing cloud + normal extraction from the TSDF volume, sm_90a.
// Replaces FullScan6 / ExtractNormals of the reference (kfusion/src/cuda/tsdf_volume.cu:486-831).
//
// The reference appends points through one global atomicAdd cursor, so its output ORDER is nondeterministic (and the
// warp nodes are picked from that order, warp_field.cpp:49-51).  Here extraction is deterministic: a counting pass,
// an exclusive scan over block counts and an emit pass produce the points in ascending (z, y, x) voxel order, +x,+y,+z
// edge within a voxel -- the same order the CPU oracle uses, so the result is comparable element by element.
//
// Work decomposition: the volume walk of volscan.cuh.  A quad whose voxels are all unobserved (W == 0) or free space (F == 1) needs
// nothing else -- on real scenes that is >90 % of them; only surface quads fetch the +x / +y / +z neighbours (L1/L2 hits).  Kernels:
// count (per-block point counts) -> scan_block_counts -> emit (the points of the blocks that have any, at their scanned offsets).  With an
// activity map the quads of inactive stretches are not loaded at all.
#include "volscan.cuh"

using namespace dfb;

namespace {

struct ExtractParams : VolumeWalk {
    float3 vs;
    Aff pose;
};

// the thread's quad i: its VX voxels (one 16-byte load when VX = 4), zeros when the quad is skipped
template <int VX>
__device__ __forceinline__ void load_quad(const ExtractParams &p, size_t v0, uint32_t (&own)[VX])
{
#pragma unroll
    for (int j = 0; j < VX; ++j) own[j] = 0u;
    if (quad_skipped(p, v0)) return;                                  // an inactive stretch cannot hold surface: not even loaded
    if (VX == 4) {
        const uint4 q = __ldg(reinterpret_cast<const uint4 *>(p.data + v0));
        own[0] = q.x; own[1 % VX] = q.y; own[2 % VX] = q.z; own[3 % VX] = q.w;
    } else {
        own[0] = __ldg(p.data + v0);
    }
}

// Calls emit(point) for every zero crossing owned by the quad at v0, in (voxel, axis) order.
template <int VX, typename Emit>
__device__ __forceinline__ void thread_crossings(const ExtractParams &p, size_t v0, const uint32_t (&own)[VX], Emit emit)
{
    bool any = false;
#pragma unroll
    for (int j = 0; j < VX; ++j) any |= vox_active(own[j]);
    if (!any) return;
    const QuadCoord c = quad_coord(p, v0);
    if (c.z >= p.Dz - 1) return;                                      // voxel_crossings' bounds, tested before the geometry
    const size_t slice = (size_t)p.Dx * p.Dy;
#pragma unroll
    for (int j = 0; j < VX; ++j) {
        if (!vox_active(own[j])) continue;
        const float F = vox_f(own[j]);
        const float3 V = make_float3(((float)(c.x0 + j) + 0.5f) * p.vs.x, ((float)c.y + 0.5f) * p.vs.y, ((float)c.z + 0.5f) * p.vs.z);
        voxel_crossings(p, own[j], c.x0 + j, c.y, c.z,
                        [&](int a) {
                            if (a == 0) return (j + 1 < VX) ? own[(j + 1) % VX] : __ldg(p.data + v0 + VX);
                            return __ldg(p.data + v0 + j + (a == 1 ? (size_t)p.Dx : slice));
                        },
                        [&](int a, float Fn) {                         // the crossing, interpolated between the two voxel centres
                            const float d_inv = 1.f / (fabsf(F) + fabsf(Fn));
                            float3 q = V;
                            if (a == 0) q.x = (V.x * fabsf(Fn) + (V.x + p.vs.x) * fabsf(F)) * d_inv;
                            else if (a == 1) q.y = (V.y * fabsf(Fn) + (V.y + p.vs.y) * fabsf(F)) * d_inv;
                            else q.z = (V.z * fabsf(Fn) + (V.z + p.vs.z) * fabsf(F)) * d_inv;
                            emit(aff_mul(p.pose, q));
                        });
    }
}

template <int VX>
__device__ __forceinline__ int quad_count(const ExtractParams &p, size_t v0, const uint32_t (&own)[VX])
{
    int n = 0;
    thread_crossings<VX>(p, v0, own, [&](const float3) { ++n; });
    return n;
}

// all of the thread's 16-byte loads are issued before any of them is used
template <int VX>
__device__ __forceinline__ void load_block_quads(const ExtractParams &p, uint32_t (&own)[WALK_QPT][VX])
{
#pragma unroll
    for (int i = 0; i < WALK_QPT; ++i) load_quad<VX>(p, quad_voxel<VX>(i), own[i]);
}

template <int VX>
__global__ void __launch_bounds__(WALK_THREADS) extract_count_kernel(const ExtractParams p, int *block_counts)
{
    DF_PDL_ENTRY();
    uint32_t own[WALK_QPT][VX];
    load_block_quads<VX>(p, own);
    int n = 0;
#pragma unroll
    for (int i = 0; i < WALK_QPT; ++i) n += quad_count<VX>(p, quad_voxel<VX>(i), own[i]);
    const int any = __syncthreads_or(n);
    if (!any) { if (threadIdx.x == 0) block_counts[blockIdx.x] = 0; return; }
    int total;
    block_exclusive_scan<WALK_THREADS>(n, &total);
    if (threadIdx.x == 0) block_counts[blockIdx.x] = total;
}

template <int VX>
__global__ void __launch_bounds__(WALK_THREADS) extract_emit_kernel(const ExtractParams p, const BlockScan scan, float4 *out, int capacity)
{
    DF_PDL_ENTRY();
    if (scan.counts[blockIdx.x] == 0) return;
    uint32_t own[WALK_QPT][VX];
    load_block_quads<VX>(p, own);
    int run = scan.base(blockIdx.x);
#pragma unroll
    for (int i = 0; i < WALK_QPT; ++i) {                              // points leave in quad order i * WALK_THREADS + tid
        const size_t v0 = quad_voxel<VX>(i);
        const int c = quad_count<VX>(p, v0, own[i]);
        int total;
        int k = run + block_exclusive_scan<WALK_THREADS>(c, &total);
        if (c)
            thread_crossings<VX>(p, v0, own[i], [&](const float3 q) {
                if (k < capacity) out[k] = make_float4(q.x, q.y, q.z, 0.f);
                ++k;
            });
        run += total;
    }
}

}  // namespace

extern "C" size_t df_extract_workspace_bytes(df_volume vol)
{
    const size_t nvox = (size_t)vol.dims[0] * vol.dims[1] * vol.dims[2];
    const size_t nblocks = (nvox + WALK_THREADS - 1) / WALK_THREADS;      // upper bound (VX = 1)
    return (block_scan_ints(nblocks) + 64) * sizeof(int);
}

extern "C" int df_extract_cloud(df_volume vol, df_aff3f pose, float *out_points, int capacity, int *count, void *workspace, void *stream)
{
    return df_extract_cloud_tracked(vol, pose, out_points, capacity, count, workspace, nullptr, stream);
}

extern "C" int df_extract_cloud_tracked(df_volume vol, df_aff3f pose, float *out_points, int capacity, int *count, void *workspace,
                                        const unsigned char *activity, void *stream)
{
    const ExtractParams p{volume_walk(vol, activity), make_float3(vol.voxel_size[0], vol.voxel_size[1], vol.voxel_size[2]), make_aff(pose)};
    const BlockScan scan = block_scan_at((int *)workspace, p.nblocks);
    cudaStream_t s = (cudaStream_t)stream;
    if (p.vx == 4) launch_pdl(extract_count_kernel<4>, dim3(p.nblocks), dim3(WALK_THREADS), 0, s, p, scan.counts);
    else launch_pdl(extract_count_kernel<1>, dim3(p.nblocks), dim3(WALK_THREADS), 0, s, p, scan.counts);
    DF_LAUNCH_CHECK();
    if (int st = scan_block_counts(scan, p.nblocks, capacity, count, s)) return st;   // > 2^20 blocks (volume > 1024^3 voxels)
    if (p.vx == 4) launch_pdl(extract_emit_kernel<4>, dim3(p.nblocks), dim3(WALK_THREADS), 0, s, p, scan, (float4 *)out_points, capacity);
    else launch_pdl(extract_emit_kernel<1>, dim3(p.nblocks), dim3(WALK_THREADS), 0, s, p, scan, (float4 *)out_points, capacity);
    DF_LAUNCH_CHECK();
    return 0;
}

// ------------------------------------------------------------------------------------------------------------------
// extract normals: reference ExtractNormals::operator() tsdf_volume.cu:714-795 (launched with 8x redundant threads,
// :817-831); here one thread per point, count optionally read from device memory.
namespace {
struct NormalsParams {
    const uint32_t *data;
    int Dx, Dy, Dz;
    float3 vs_inv, gd;
    Aff pose;
    Mat3 Rinv;
    const float4 *points;
    int n;
    const int *count_dev;
    float4 *out;
};

__device__ __forceinline__ float en_tsdf(const NormalsParams &p, int x, int y, int z)
{ return half_bits_to_float((unsigned short)(__ldg(p.data + x + (size_t)p.Dx * y + (size_t)p.Dx * p.Dy * z) & 0xffffu)); }

__device__ __forceinline__ float en_interpolate(const NormalsParams &p, const float3 cf)
{
    const float fx = floorf(cf.x), fy = floorf(cf.y), fz = floorf(cf.z);
    if (!(fx >= 0) || !(fy >= 0) || !(fz >= 0) || !(fx < (float)(p.Dx - 1)) || !(fy < (float)(p.Dy - 1)) || !(fz < (float)(p.Dz - 1)))
        return qnan();
    const int gx = (int)fx, gy = (int)fy, gz = (int)fz;
    const float a = cf.x - (float)gx, b = cf.y - (float)gy, c = cf.z - (float)gz;
    const float v000 = en_tsdf(p, gx, gy, gz), v001 = en_tsdf(p, gx, gy, gz + 1);
    const float v010 = en_tsdf(p, gx, gy + 1, gz), v011 = en_tsdf(p, gx, gy + 1, gz + 1);
    const float v100 = en_tsdf(p, gx + 1, gy, gz), v101 = en_tsdf(p, gx + 1, gy, gz + 1);
    const float v110 = en_tsdf(p, gx + 1, gy + 1, gz), v111 = en_tsdf(p, gx + 1, gy + 1, gz + 1);
    float tsdf = 0.f;
    tsdf += v000 * (1 - a) * (1 - b) * (1 - c);
    tsdf += v001 * (1 - a) * (1 - b) * c;
    tsdf += v010 * (1 - a) * b * (1 - c);
    tsdf += v011 * (1 - a) * b * c;
    tsdf += v100 * a * (1 - b) * (1 - c);
    tsdf += v101 * a * (1 - b) * c;
    tsdf += v110 * a * b * (1 - c);
    tsdf += v111 * a * b * c;
    return tsdf;
}

__global__ void __launch_bounds__(256) extract_normals_kernel(const NormalsParams p)
{
    DF_PDL_ENTRY();
    const int n = p.count_dev ? min(*p.count_dev, p.n) : p.n;
    for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < n; idx += gridDim.x * blockDim.x) {
        const float nanv = qnan();
        float3 nrm = make_float3(nanv, nanv, nanv);
        const float4 pt = p.points[idx];
        const float3 point = mat3_mul(p.Rinv, sub3(make_float3(pt.x, pt.y, pt.z), p.pose.t));
        const int gx = __float2int_rn(point.x * p.vs_inv.x), gy = __float2int_rn(point.y * p.vs_inv.y), gz = __float2int_rn(point.z * p.vs_inv.z);
        if (gx > 1 && gy > 1 && gz > 1 && gx < p.Dx - 2 && gy < p.Dy - 2 && gz < p.Dz - 2) {
            float3 t;
            t = point; t.x += p.gd.x; const float Fx1 = en_interpolate(p, mul3(t, p.vs_inv));
            t = point; t.x -= p.gd.x; const float Fx2 = en_interpolate(p, mul3(t, p.vs_inv));
            nrm.x = (Fx1 - Fx2) / p.gd.x;
            t = point; t.y += p.gd.y; const float Fy1 = en_interpolate(p, mul3(t, p.vs_inv));
            t = point; t.y -= p.gd.y; const float Fy2 = en_interpolate(p, mul3(t, p.vs_inv));
            nrm.y = (Fy1 - Fy2) / p.gd.y;
            t = point; t.z += p.gd.z; const float Fz1 = en_interpolate(p, mul3(t, p.vs_inv));
            t = point; t.z -= p.gd.z; const float Fz2 = en_interpolate(p, mul3(t, p.vs_inv));
            nrm.z = (Fz1 - Fz2) / p.gd.z;
            nrm = normalized3(mat_mul(p.pose.r0, p.pose.r1, p.pose.r2, nrm));
        }
        p.out[idx] = make_float4(nrm.x, nrm.y, nrm.z, 0.f);
    }
}
}  // namespace

extern "C" int df_extract_normals(df_volume vol, const float *points, int n_points, const int *count_dev, df_aff3f pose,
                                  const float *Rinv_host9, float delta_factor, float *out_normals, void *stream)
{
    if (n_points <= 0) return 0;
    NormalsParams p;
    p.data = vol.data;
    p.Dx = vol.dims[0]; p.Dy = vol.dims[1]; p.Dz = vol.dims[2];
    p.vs_inv = make_float3(1.f / vol.voxel_size[0], 1.f / vol.voxel_size[1], 1.f / vol.voxel_size[2]);
    p.gd = make_float3(vol.voxel_size[0] * delta_factor, vol.voxel_size[1] * delta_factor, vol.voxel_size[2] * delta_factor);
    p.pose = make_aff(pose);
    p.Rinv = make_mat3(Rinv_host9);
    p.points = (const float4 *)points; p.n = n_points; p.count_dev = count_dev; p.out = (float4 *)out_normals;
    const int blocks = count_dev ? DF_NUM_SMS * 8 : div_up(n_points, 256);
    launch_pdl(extract_normals_kernel, dim3(blocks), dim3(256), 0, (cudaStream_t)stream, p);
    DF_LAUNCH_CHECK();
    return 0;
}
