// extend.cu -- extending the warp field on sm_90a (SURVEY.md 8f(3)).
//
// The reference describes this step and never wrote it (Report.md, "4. Extending the warp field - stubbed out functionality": "As the
// canonical model grows with new data being fused in, the warp field needs to grow as well, to support it").  It is assembled here from
// the pieces the reference does define; the CPU restatement it is tested against is oracle/orc_fusion.c (orc_extend_field):
//   * a point of the extracted canonical cloud is UNSUPPORTED when its nearest node (WarpField::KNN, warp_field.cpp:247-251) is farther
//     than `radius` (float d^2 > radius*radius); NaN points are skipped;
//   * the unsupported points are subsampled the way WarpField::init subsamples the first cloud (every step-th, warp_field.cpp:49-60), in
//     cloud order -- deterministic here because df_extract_cloud emits in (z, y, x, axis) order;
//   * each becomes a node as init makes them (:68-80): identity DualQuaternion(), weight 3; appended until max_nodes.
// Three launches: nearest-node test + per-block counts, a one-block exclusive scan (which also publishes the new node count), and the
// append (ballot ranks inside the block).  The caller rebuilds the node grid (df_build_node_grid) when the count has changed.
#include "warp_common.cuh"
#include "volscan.cuh"

using namespace dfb;

namespace {

__device__ __forceinline__ bool extend_unsupported(const float *__restrict__ nodes, int M, const void *grid, KnnSmem &sm, const float *__restrict__ cloud,
                                                   int q, int n, int stride, float r2, float3 &pt)
{
    bool valid = false;
    pt = make_float3(0.f, 0.f, 0.f);
    if (q < n) {
        const float *p = cloud + (size_t)q * stride;
        pt = make_float3(p[0], p[1], p[2]);
        valid = !(isnan(pt.x) || isnan(pt.y) || isnan(pt.z));
    }
    int bi[8]; float bd[8];
    if (grid) knn8_grid(grid, valid, pt.x, pt.y, pt.z, bi, bd);
    else knn8_scan(nodes, M, valid, pt.x, pt.y, pt.z, sm, bi, bd);
    return valid && bd[0] > r2;
}

__global__ void __launch_bounds__(256) extend_count_kernel(const float *__restrict__ nodes, int M, const void *__restrict__ grid, const float *__restrict__ cloud,
                                                           int capacity, const int *__restrict__ count_dev, int stride, float r2, int *block_count,
                                                           unsigned char *flags)
{
    DF_PDL_ENTRY();
    __shared__ KnnSmem sm;
    const int n = count_dev ? min(*count_dev, capacity) : capacity;
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    float3 pt;
    const bool u = extend_unsupported(nodes, M, grid, sm, cloud, q, n, stride, r2, pt);
    if (q < capacity) flags[q] = u ? 1 : 0;
    const int c = __syncthreads_count(u);
    if (threadIdx.x == 0) block_count[blockIdx.x] = c;
}

// exclusive scan of the block counts in place; M_out = min(max_nodes, M + ceil(total / step))
__global__ void __launch_bounds__(1024) extend_scan_kernel(int *block_count, int nblocks, int M, int max_nodes, int step, int *M_out)
{
    DF_PDL_ENTRY();
    const int total = block_scan_in_place(block_count, nblocks);
    if (threadIdx.x == 0) {
        const long long want = (long long)M + ((long long)total + step - 1) / step;
        *M_out = (int)(want < (long long)max_nodes ? want : (long long)max_nodes);
        if (*M_out < M) *M_out = M;
    }
}

__global__ void __launch_bounds__(256) extend_append_kernel(float *nodes, int M, int max_nodes, const float *__restrict__ cloud, int capacity, int stride, int step,
                                                            const int *__restrict__ block_offset, const unsigned char *__restrict__ flags)
{
    DF_PDL_ENTRY();
    __shared__ int warp_count[8];
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    const bool u = q < capacity && flags[q] != 0;
    const unsigned ballot = __ballot_sync(0xffffffffu, u);
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    if (lane == 0) warp_count[w] = __popc(ballot);
    __syncthreads();
    if (!u) return;
    int rank = block_offset[blockIdx.x] + __popc(ballot & ((1u << lane) - 1u));
    for (int i = 0; i < w; ++i) rank += warp_count[i];
    if (rank % step != 0) return;
    const long long slot = (long long)M + rank / step;
    if (slot >= max_nodes) return;
    const float *p = cloud + (size_t)q * stride;
    float4 *n4 = reinterpret_cast<float4 *>(nodes + (size_t)slot * DF_NODE_STRIDE);
    n4[0] = make_float4(p[0], p[1], p[2], 1.f);          // vertex, rotation w
    n4[1] = make_float4(0.f, 0.f, 0.f, 1.f);             // rotation xyz, dual w   (DualQuaternion(): rotation (1,0,0,0), dual (1,0,0,0))
    n4[2] = make_float4(0.f, 0.f, 0.f, 3.f);             // dual xyz, weight = 3 * voxel_size with voxel_size forced to 1 (warp_field.cpp:48,76)
}

}  // namespace

extern "C" size_t df_extend_field_workspace_bytes(int capacity)
{
    return (size_t)(div_up(capacity > 0 ? capacity : 1, 256) + 16) * sizeof(int) + (size_t)(capacity > 0 ? capacity : 1) + 64;
}

extern "C" int df_extend_field(float *nodes, int M, int max_nodes, const void *node_grid, const float *cloud, int capacity, const int *count_dev,
                               int stride, float radius, int step, int *M_out_dev, void *workspace, void *stream)
{
    if (!nodes || !cloud || !M_out_dev || !workspace || M <= 0 || capacity <= 0 || step <= 0 || stride < 3) return (int)cudaErrorInvalidValue;
    cudaStream_t s = (cudaStream_t)stream;
    const int nblocks = div_up(capacity, 256);
    int *block_count = (int *)workspace;
    unsigned char *flags = (unsigned char *)(block_count + nblocks + 16);
    launch_pdl(extend_count_kernel, dim3(nblocks), dim3(256), 0, s, (const float *)nodes, M, node_grid, cloud, capacity, count_dev, stride, radius * radius,
               block_count, flags);
    launch_pdl(extend_scan_kernel, dim3(1), dim3(1024), 0, s, block_count, nblocks, M, max_nodes, step, M_out_dev);
    launch_pdl(extend_append_kernel, dim3(nblocks), dim3(256), 0, s, nodes, M, max_nodes, cloud, capacity, stride, step, (const int *)block_count,
               (const unsigned char *)flags);
    DF_LAUNCH_CHECK();
    return 0;
}
