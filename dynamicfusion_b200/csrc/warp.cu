// warp.cu -- fused k-NN + node weights + dual-quaternion-blend warp of vertex/normal sets on sm_90a.
// Replaces WarpField::KNN / getWeightsAndUpdateKNN / DQB / warp of the reference (kfusion/src/warp_field.cpp:180-251),
// which run single-threaded on the CPU through a nanoflann kd-tree (~1 M queries per frame, the reference's dominant
// cost, SURVEY.md section 3.4).  The node table (M x 48 B) is GPU-resident; a block stages node positions tile by tile
// in shared memory and every thread scans them for its own point.
#include "warp_common.cuh"
#include "volscan.cuh"

using namespace dfb;

namespace {

__global__ void __launch_bounds__(256) knn8_kernel(const float *__restrict__ nodes, int M, const void *__restrict__ grid,
                                                   const float *__restrict__ queries, int N,
                                                   int qstride, int *__restrict__ idx, float *__restrict__ d2)
{
    DF_PDL_ENTRY();
    __shared__ KnnSmem sm;
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    float qx = 0.f, qy = 0.f, qz = 0.f;
    bool valid = false;
    if (q < N) {
        const float *p = queries + (size_t)q * qstride;
        qx = p[0]; qy = p[1]; qz = p[2];
        valid = !(isnan(qx) || isnan(qy) || isnan(qz));
    }
    int bi[8]; float bd[8];
    if (grid) knn8_grid(grid, valid, qx, qy, qz, bi, bd);
    else knn8_scan(nodes, M, valid, qx, qy, qz, sm, bi, bd);
    if (q < N) {
#pragma unroll
        for (int i = 0; i < 8; ++i) { idx[(size_t)q * 8 + i] = bi[i]; d2[(size_t)q * 8 + i] = bd[i]; }
    }
}

struct WarpParams {
    const float *nodes; int M; const void *grid;
    float *points; float *normals; int N; int stride;
    Aff w2l;
    int flags;
    int *idx; float *w;       // neighbours / weights: outputs, or inputs when DF_WARP_REUSE_KNN
    int cols;                 // > 0: the points are an image of that many columns (DF_WARP_IMAGE_COLS): warps take 8 x 4 pixel patches
};

// cv::Affine3f * Vec3f (opencv2/core/affine.hpp): m0*x + m1*y + m2*z + m3 evaluated left to right
__device__ __forceinline__ float3 aff_apply_cv(const Aff &a, const float3 v)
{
    return make_float3(a.r0.x * v.x + a.r0.y * v.y + a.r0.z * v.z + a.t.x,
                       a.r1.x * v.x + a.r1.y * v.y + a.r1.z * v.z + a.t.y,
                       a.r2.x * v.x + a.r2.y * v.y + a.r2.z * v.z + a.t.z);
}

// WarpField::warp, warp_field.cpp:180-195.  kReuse: neighbours and weights of these very points were computed by an
// earlier pass (the data-term solve queries the same warped vertices, CombinedSolver.h:66-84) and are read back instead
// of being searched again.
template <bool kReuse>
__global__ void __launch_bounds__(256) warp_kernel(const WarpParams p)
{
    DF_PDL_ENTRY();
    __shared__ KnnSmem sm;
    const int q = kReuse ? (int)(blockIdx.x * blockDim.x + threadIdx.x) : patch_vertex(blockIdx.x, threadIdx.x, p.cols);
    float3 pt = make_float3(0.f, 0.f, 0.f), nr = pt;
    bool valid = false;
    if (q < p.N) {
        const float *pp = p.points + (size_t)q * p.stride;
        pt = make_float3(pp[0], pp[1], pp[2]);
        valid = !isnan(pt.x);
        if (valid) {
            const float *np = p.normals + (size_t)q * p.stride;
            nr = make_float3(np[0], np[1], np[2]);
            valid = !isnan(nr.x);
        }
    }
    int bi[8]; float bd[8]; float w8[8];
    if (kReuse) {
        if (q >= p.N) return;
        const int4 ia = *reinterpret_cast<const int4 *>(p.idx + (size_t)q * 8), ib = *reinterpret_cast<const int4 *>(p.idx + (size_t)q * 8 + 4);
        const float4 wa = *reinterpret_cast<const float4 *>(p.w + (size_t)q * 8), wb = *reinterpret_cast<const float4 *>(p.w + (size_t)q * 8 + 4);
        bi[0] = ia.x; bi[1] = ia.y; bi[2] = ia.z; bi[3] = ia.w; bi[4] = ib.x; bi[5] = ib.y; bi[6] = ib.z; bi[7] = ib.w;
        w8[0] = wa.x; w8[1] = wa.y; w8[2] = wa.z; w8[3] = wa.w; w8[4] = wb.x; w8[5] = wb.y; w8[6] = wb.z; w8[7] = wb.w;
#pragma unroll
        for (int i = 0; i < 8; ++i) bd[i] = 0.f;
        valid = valid && bi[0] >= 0;          // rows the earlier pass skipped (NaN) carry idx = -1
    } else {
        if (p.grid) knn8_grid(p.grid, valid, pt.x, pt.y, pt.z, bi, bd);
        else knn8_scan(p.nodes, p.M, valid, pt.x, pt.y, pt.z, sm, bi, bd);
        if (q >= p.N) return;
    }
    if (valid) {
        const Dqb d = dqb_blend<kReuse>(p.nodes, bi, bd, w8);
        const float3 wp = aff_apply_cv(p.w2l, dq_transform(d, pt));
        float3 wn;
        if (p.flags & DF_WARP_NORMAL_ROTATE_ONLY) {
            const float3 r = qrotate(d.rot, nr);
            wn = make_float3(p.w2l.r0.x * r.x + p.w2l.r0.y * r.y + p.w2l.r0.z * r.z,
                             p.w2l.r1.x * r.x + p.w2l.r1.y * r.y + p.w2l.r1.z * r.z,
                             p.w2l.r2.x * r.x + p.w2l.r2.y * r.y + p.w2l.r2.z * r.z);
        } else {
            wn = aff_apply_cv(p.w2l, dq_transform(d, nr));       // the reference also translates normals
        }
        float *pp = p.points + (size_t)q * p.stride;
        pp[0] = wp.x; pp[1] = wp.y; pp[2] = wp.z;
        float *np = p.normals + (size_t)q * p.stride;
        np[0] = wn.x; np[1] = wn.y; np[2] = wn.z;
    } else if (!kReuse) {
#pragma unroll
        for (int i = 0; i < 8; ++i) w8[i] = 0.f;
    }
    if (!kReuse && p.idx) {
#pragma unroll
        for (int i = 0; i < 8; ++i) { p.idx[(size_t)q * 8 + i] = bi[i]; p.w[(size_t)q * 8 + i] = w8[i]; }
    }
}

// ------------------------------------------------------------------------------------------------------------------
// DF_WARP_REF_NORMAL_INDEX: the reference's normal cursor (warp_field.cpp:182-194).  `i` advances only after a point has been
// warped, and a point is skipped when ITS x is NaN or when normals[i] is NaN -- so the j-th non-NaN point is paired with normal j, and
// once the cursor reaches the first NaN normal (index c) it never moves again: points of rank >= c are left untouched.  In parallel:
// c = the smallest index of a NaN normal (one atomicMin), rank = exclusive count of non-NaN points (block counts -> one-block scan ->
// ballot ranks inside the warp kernel).  Every rank is unique, so no two threads touch the same normal.
__global__ void __launch_bounds__(256) warp_cursor_count_kernel(const float *__restrict__ points, const float *__restrict__ normals, int N, int stride,
                                                                int *block_count, int *first_nan_normal)
{
    DF_PDL_ENTRY();
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    const bool valid = q < N && !isnan(points[(size_t)q * stride]);
    const int n = __syncthreads_count(valid);
    if (threadIdx.x == 0) block_count[blockIdx.x] = n;
    if (q < N && isnan(normals[(size_t)q * stride])) atomicMin(first_nan_normal, q);
}

__global__ void __launch_bounds__(1024) warp_cursor_scan_kernel(int *block_count, int nblocks)
{
    DF_PDL_ENTRY();
    block_scan_in_place(block_count, nblocks);
}

__global__ void __launch_bounds__(256) warp_cursor_kernel(const WarpParams p, const int *__restrict__ block_offset, const int *__restrict__ first_nan_normal)
{
    DF_PDL_ENTRY();
    __shared__ KnnSmem sm;
    __shared__ int warp_count[8];
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    float3 pt = make_float3(0.f, 0.f, 0.f);
    bool valid = false;
    if (q < p.N) {
        const float *pp = p.points + (size_t)q * p.stride;
        pt = make_float3(pp[0], pp[1], pp[2]);
        valid = !isnan(pt.x);
    }
    const unsigned ballot = __ballot_sync(0xffffffffu, valid);
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    if (lane == 0) warp_count[w] = __popc(ballot);
    __syncthreads();
    int rank = block_offset[blockIdx.x] + __popc(ballot & ((1u << lane) - 1u));
    for (int i = 0; i < w; ++i) rank += warp_count[i];
    valid = valid && rank < *first_nan_normal;
    int bi[8]; float bd[8];
    if (p.grid) knn8_grid(p.grid, valid, pt.x, pt.y, pt.z, bi, bd);
    else knn8_scan(p.nodes, p.M, valid, pt.x, pt.y, pt.z, sm, bi, bd);
    if (!valid) return;
    float *np = p.normals + (size_t)rank * p.stride;
    const float3 nr = make_float3(np[0], np[1], np[2]);
    const Dqb d = dqb_blend<false>(p.nodes, bi, bd, nullptr);
    const float3 wp = aff_apply_cv(p.w2l, dq_transform(d, pt));
    float3 wn;
    if (p.flags & DF_WARP_NORMAL_ROTATE_ONLY) {
        const float3 r = qrotate(d.rot, nr);
        wn = make_float3(p.w2l.r0.x * r.x + p.w2l.r0.y * r.y + p.w2l.r0.z * r.z,
                         p.w2l.r1.x * r.x + p.w2l.r1.y * r.y + p.w2l.r1.z * r.z,
                         p.w2l.r2.x * r.x + p.w2l.r2.y * r.y + p.w2l.r2.z * r.z);
    } else {
        wn = aff_apply_cv(p.w2l, dq_transform(d, nr));
    }
    float *pp = p.points + (size_t)q * p.stride;
    pp[0] = wp.x; pp[1] = wp.y; pp[2] = wp.z;
    np[0] = wn.x; np[1] = wn.y; np[2] = wn.z;
}

}  // namespace

extern "C" int df_knn8(const float *nodes, int M, const void *node_grid, const float *queries, int N, int qstride, int32_t *idx, float *d2,
                       void *stream)
{
    if (N <= 0) return 0;
    launch_pdl(knn8_kernel, dim3(div_up(N, 256)), dim3(256), 0, (cudaStream_t)stream, nodes, M, node_grid, queries, N, qstride, idx, d2);
    DF_LAUNCH_CHECK();
    return 0;
}

extern "C" int df_warp(const float *nodes, int M, const void *node_grid, float *points, float *normals, int N, int stride,
                       df_aff3f warp_to_live, int flags, int32_t *idx, float *w, void *stream)
{
    if (N <= 0) return 0;
    if (flags & DF_WARP_REF_NORMAL_INDEX) {
        // the reference's normal cursor (warp_field.cpp:182-194); neighbour output / re-use is not offered on this path
        if ((flags & DF_WARP_REUSE_KNN) || idx || w) return (int)cudaErrorNotSupported;
        cudaStream_t s = (cudaStream_t)stream;
        const int nblocks = div_up(N, 256);
        int *scratch = nullptr;
        cudaError_t e = cudaMallocAsync((void **)&scratch, (size_t)(nblocks + 1) * sizeof(int), s);
        if (e != cudaSuccess) return (int)e;
        e = cudaMemcpyAsync(scratch + nblocks, &N, sizeof(int), cudaMemcpyHostToDevice, s);      // first NaN normal: N = none (pageable source: copied before return)
        if (e != cudaSuccess) { cudaFreeAsync(scratch, s); return (int)e; }
        WarpParams p;
        p.nodes = nodes; p.M = M; p.grid = node_grid; p.points = points; p.normals = normals; p.N = N; p.stride = stride;
        p.w2l = make_aff(warp_to_live); p.flags = flags; p.idx = nullptr; p.w = nullptr; p.cols = 0;
        launch_pdl(warp_cursor_count_kernel, dim3(nblocks), dim3(256), 0, s, (const float *)points, (const float *)normals, N, stride, scratch, scratch + nblocks);
        launch_pdl(warp_cursor_scan_kernel, dim3(1), dim3(1024), 0, s, scratch, nblocks);
        launch_pdl(warp_cursor_kernel, dim3(nblocks), dim3(256), 0, s, p, (const int *)scratch, (const int *)(scratch + nblocks));
        cudaFreeAsync(scratch, s);
        DF_LAUNCH_CHECK();
        return 0;
    }
    if ((flags & DF_WARP_REUSE_KNN) && (!idx || !w)) return (int)cudaErrorInvalidValue;
    WarpParams p;
    p.nodes = nodes; p.M = M; p.grid = node_grid; p.points = points; p.normals = normals; p.N = N; p.stride = stride;
    p.w2l = make_aff(warp_to_live); p.flags = flags; p.idx = idx; p.w = w;
    const int cols = (flags >> 8) & 0xffff;                      // DF_WARP_IMAGE_COLS: 8 x 4 pixel patches per warp when the shape allows it
    p.cols = (cols > 0 && N % cols == 0 && cols % 32 == 0 && (N / cols) % 8 == 0) ? cols : 0;
    if (flags & DF_WARP_REUSE_KNN) launch_pdl(warp_kernel<true>, dim3(div_up(N, 256)), dim3(256), 0, (cudaStream_t)stream, p);
    else launch_pdl(warp_kernel<false>, dim3(div_up(N, 256)), dim3(256), 0, (cudaStream_t)stream, p);
    DF_LAUNCH_CHECK();
    return 0;
}
