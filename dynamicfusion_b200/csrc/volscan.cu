// volscan.cu -- the two-level block scan of volscan.cuh (scan_block_counts), sm_90a.
#include "volscan.cuh"

using namespace dfb;

namespace {

// exclusive scan of in[0 .. n) in chunks of 1024 (one block per chunk, warp-shuffle scan) -> out; chunk total -> chunk_total[chunk],
// clamped to capacity
__global__ void __launch_bounds__(1024) scan_block_counts_kernel(const int *in, int n, int *out, int *chunk_total, int capacity)
{
    DF_PDL_ENTRY();
    __shared__ int wsum[32];
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const int i = blockIdx.x * 1024 + t;
    const int c = i < n ? in[i] : 0;
    int incl = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
    if (lane == 31) wsum[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        int w = wsum[lane];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, w, o); if (lane >= o) w += v; }
        wsum[lane] = w;
    }
    __syncthreads();
    const int base = warp ? wsum[warp - 1] : 0;
    if (i < n) out[i] = base + incl - c;
    if (t == 1023) chunk_total[blockIdx.x] = min(wsum[31], capacity);
}

}  // namespace

// the counts of each chunk of 1024 blocks, then the <= 1024 chunk totals in one block
int dfb::scan_block_counts(const BlockScan &ws, int n, int capacity, int *total, cudaStream_t s)
{
    if (!scan_fits(n)) return (int)cudaErrorInvalidValue;
    const int nsuper = (n + 1023) / 1024;
    launch_pdl(scan_block_counts_kernel, dim3(nsuper), dim3(1024), 0, s, (const int *)ws.counts, n, ws.offsets, ws.super, 0x7fffffff);
    DF_LAUNCH_CHECK();
    launch_pdl(scan_block_counts_kernel, dim3(1), dim3(1024), 0, s, (const int *)ws.super, nsuper, ws.super + 1024, total, capacity);
    DF_LAUNCH_CHECK();
    return 0;
}
