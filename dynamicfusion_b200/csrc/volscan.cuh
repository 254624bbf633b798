// volscan.cuh -- the extraction's walk over the TSDF volume, its crossing rule and its deterministic scans (sm_90a).
//
// The cloud's point order, and with it every triangle of the mesh (triangles are cloud indices), follows from the decisions made here:
// extract.cu emits the points and mesh.cu recomputes where they went, so both walk the volume through this header and nothing else.
#pragma once
#include "df_common.cuh"

namespace dfb {

// ---------------------------------------------------------------------------------------------------------------- the volume walk
// The volume is one contiguous array in (z, y, x) order cut into blocks of WALK_THREADS * WALK_QPT quads; a quad is VX consecutive
// voxels, one 16-byte load when VX = 4.  Thread t of a block owns its quads i * WALK_THREADS + t, i = 0 .. WALK_QPT - 1, so every load
// instruction of a warp is one contiguous 512-byte request.  History: one quad per thread meant 131,072 CTAs for 512^3 -- the emit pass,
// whose CTAs mostly return at once, was limited by block scheduling, not memory; one WARP per block (8 quads per lane, shuffle scans)
// removed the scheduling cost but serialised the dependent neighbour fetches of the surface quads and was slower still.
constexpr int WALK_THREADS = 256;
constexpr int WALK_QPT = 4;

struct VolumeWalk {
    const uint32_t *data;
    int Dx, Dy, Dz;
    size_t nvox;
    int nblocks, vx;
    const unsigned char *activity;   // optional (dfusion.h, DF_ACTIVITY_VOXELS): the quads of inactive stretches are skipped
};

// VX = 4 when every row starts 16-byte aligned
inline int pick_vx(const df_volume &vol) { return (vol.dims[0] % 4 == 0 && ((uintptr_t)vol.data & 15u) == 0) ? 4 : 1; }

inline VolumeWalk volume_walk(const df_volume &vol, const unsigned char *activity)
{
    VolumeWalk w;
    w.data = vol.data;
    w.Dx = vol.dims[0]; w.Dy = vol.dims[1]; w.Dz = vol.dims[2];
    w.nvox = (size_t)vol.dims[0] * vol.dims[1] * vol.dims[2];
    w.vx = pick_vx(vol);
    const size_t per_block = (size_t)WALK_THREADS * WALK_QPT * w.vx;
    w.nblocks = (int)((w.nvox + per_block - 1) / per_block);
    w.activity = activity;
    return w;
}

// first voxel of the calling thread's quad i of its block
template <int VX>
__device__ __forceinline__ size_t quad_voxel(int i)
{
    return ((size_t)blockIdx.x * WALK_THREADS * WALK_QPT + (size_t)(i * WALK_THREADS) + threadIdx.x) * VX;
}

struct QuadCoord { int x0, y, z; };
__device__ __forceinline__ QuadCoord quad_coord(const VolumeWalk &w, size_t v0)
{
    const size_t slice = (size_t)w.Dx * w.Dy;
    QuadCoord c;
    c.z = (int)(v0 / slice);
    const int rem = (int)(v0 - (size_t)c.z * slice);
    c.y = rem / w.Dx;
    c.x0 = rem - c.y * w.Dx;
    return c;
}

// past the end of the volume, or in a stretch the activity map marks inactive: such a stretch holds no active voxel, so it owns no
// point and anchors no polygonised cube (its anchor corner would be inactive)
__device__ __forceinline__ bool quad_skipped(const VolumeWalk &w, size_t v0)
{
    return v0 >= w.nvox || (w.activity && !w.activity[v0 / DF_ACTIVITY_VOXELS]);
}

// ------------------------------------------------------------------------------------------------------------- the crossing rule
__device__ __forceinline__ float vox_f(uint32_t v) { return half_bits_to_float((unsigned short)(v & 0xffffu)); }
__device__ __forceinline__ bool sign_change(float F, float Fn) { return (F > 0 && Fn < 0) || (F < 0 && Fn > 0); }

// The rule: voxel v at (x, y, z) emits a cloud point on axis a when it and its neighbour on that axis (+x, +y, +z) are active and their
// F differ in sign; the neighbour must lie inside the volume, and z < dims.z - 1 (tsdf_volume.cu:548-633, loop bound :553).
// voxel_crossings calls on(a, Fn) for each such axis in axis order, Fn the neighbour's F; nb(a) returns the neighbour on axis a and is
// called only where that neighbour lies inside the volume.
template <typename Nb, typename On>
__device__ __forceinline__ void voxel_crossings(const VolumeWalk &w, uint32_t v, int x, int y, int z, Nb nb, On on)
{
    if (!vox_active(v) || z >= w.Dz - 1) return;
    const float F = vox_f(v);
    if (x + 1 < w.Dx) {
        const uint32_t n = nb(0);
        if (vox_active(n)) { const float Fn = vox_f(n); if (sign_change(F, Fn)) on(0, Fn); }
    }
    if (y + 1 < w.Dy) {
        const uint32_t n = nb(1);
        if (vox_active(n)) { const float Fn = vox_f(n); if (sign_change(F, Fn)) on(1, Fn); }
    }
    {
        const uint32_t n = nb(2);
        if (vox_active(n)) { const float Fn = vox_f(n); if (sign_change(F, Fn)) on(2, Fn); }
    }
}

// the axes (bit a = axis a) on which voxel v at (x, y, z) emits a cloud point, given its +x, +y, +z neighbours nx, ny, nz
__device__ __forceinline__ int crossing_axes(const VolumeWalk &w, uint32_t v, uint32_t nx, uint32_t ny, uint32_t nz, int x, int y, int z)
{
    int f = 0;
    voxel_crossings(w, v, x, y, z, [&](int a) { return a == 0 ? nx : (a == 1 ? ny : nz); }, [&](int a, float) { f |= 1 << a; });
    return f;
}

// ------------------------------------------------------------------------------------------------------------------ the scans
// exclusive scan of v over a block of THREADS threads; *total (if given) receives the block's sum.  Every thread must call it.
template <int THREADS>
__device__ __forceinline__ int block_exclusive_scan(int v, int *total)
{
    __shared__ int warp_sums[THREADS / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int n = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += n;
    }
    if (lane == 31) warp_sums[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        int w = lane < THREADS / 32 ? warp_sums[lane] : 0;
#pragma unroll
        for (int o = 1; o < THREADS / 32; o <<= 1) {
            const int n = __shfl_up_sync(0xffffffffu, w, o);
            if (lane >= o) w += n;
        }
        if (lane < THREADS / 32) warp_sums[lane] = w;
    }
    __syncthreads();
    const int base = warp ? warp_sums[warp - 1] : 0;
    if (total) *total = warp_sums[THREADS / 32 - 1];
    __syncthreads();
    return base + incl - v;
}

// Workspace of scan_block_counts over n per-block counts: block_scan_ints(n) ints, counts first.  The exclusive prefix of block b is
// base(b): the prefix of its chunk of 1024 blocks plus its offset inside the chunk.  (A single-block serial-chunk scan of the 131,072
// counts of a 512^3 volume is a long serial chain.)
struct BlockScan {
    int *counts;    // [n], written by the caller's count pass
    int *offsets;   // [n] exclusive prefix inside the chunk
    int *super;     // [2048] chunk totals, then from 1024 on their exclusive prefix
    __device__ __forceinline__ int base(int b) const { return super[1024 + (b >> 10)] + offsets[b]; }
};
inline size_t block_scan_ints(size_t n) { return 2 * n + 2048; }
inline BlockScan block_scan_at(int *ws, int n) { return {ws, ws + n, ws + 2 * (size_t)n}; }
inline bool scan_fits(int nblocks) { return nblocks <= 1024 * 1024; }

// Deterministic two-level exclusive scan of ws.counts[0 .. n); *total (device) receives min(sum, capacity).  Two launches.  volscan.cu
int scan_block_counts(const BlockScan &ws, int n, int capacity, int *total, cudaStream_t s);

// Exclusive scan of a[0 .. n) in place by one block of 1024 threads, 1024 entries at a time; returns the sum.  Every thread must call it.
__device__ __forceinline__ int block_scan_in_place(int *a, int n)
{
    __shared__ int sm[1024];
    __shared__ int carry;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (int base = 0; base < n; base += 1024) {
        const int i = base + threadIdx.x;
        const int v = i < n ? a[i] : 0;
        sm[threadIdx.x] = v;
        __syncthreads();
        for (int o = 1; o < 1024; o <<= 1) {
            const int t = threadIdx.x >= o ? sm[threadIdx.x - o] : 0;
            __syncthreads();
            sm[threadIdx.x] += t;
            __syncthreads();
        }
        if (i < n) a[i] = carry + sm[threadIdx.x] - v;
        __syncthreads();
        if (threadIdx.x == 1023) carry += sm[1023];
        __syncthreads();
    }
    return carry;
}

}  // namespace dfb
