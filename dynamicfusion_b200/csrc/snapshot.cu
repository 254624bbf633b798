// snapshot.cu -- brick packing of a TSDF volume for snapshots (df_volume_pack_* / df_volume_unpack, dfusion.h), sm_90a.
//
// The volume is cut into DF_BRICK^3 bricks (the activity map's brick table, brick (bx, by, bz) at ((bz * nby) + by) * nbx + bx).  Each brick
// is empty (every in-volume voxel 0, what df_clear_volume writes), uniform (every in-volume voxel the same non-zero word: free space) or
// mixed.  A packed volume is one class byte per brick plus a payload of u32 words in brick order: nothing for an empty brick, its word for
// a uniform one, its 512 words in (z, y, x) order for a mixed one (slots outside the volume written as 0).  No offsets are stored; both
// directions derive them with the deterministic block scan of volscan.cuh (scan_block_counts).
//
// Work decomposition: one warp per brick, PK_WARPS bricks (consecutive in brick order) per block.  Lane l loads quads l, l + 32, l + 64,
// l + 96 of the brick (quad j = row j >> 1 = (z, y) = (j >> 4, (j >> 1) & 7), x half j & 1): every 32-byte row of the brick is one sector,
// and the four 16-byte loads of a lane are independent.
#include "volscan.cuh"

using namespace dfb;

namespace {

constexpr int PK_WARPS = 8;
constexpr int PK_THREADS = PK_WARPS * 32;
constexpr int BRICK_WORDS = DF_BRICK * DF_BRICK * DF_BRICK;
static_assert(DF_BRICK == 8, "the lane -> quad mapping assumes 8^3 bricks");

struct PackGeom {
    int Dx, Dy, Dz;
    int nbx, nby, nbz;
    int nbricks, nblocks;
};

PackGeom geom_of(const df_volume &v)
{
    PackGeom g;
    g.Dx = v.dims[0]; g.Dy = v.dims[1]; g.Dz = v.dims[2];
    g.nbx = (g.Dx + DF_BRICK - 1) / DF_BRICK; g.nby = (g.Dy + DF_BRICK - 1) / DF_BRICK; g.nbz = (g.Dz + DF_BRICK - 1) / DF_BRICK;
    g.nbricks = g.nbx * g.nby * g.nbz;
    g.nblocks = (g.nbricks + PK_WARPS - 1) / PK_WARPS;
    return g;
}

// dims[0] % 32 == 0 (every brick row lies inside the volume in x, and is 16-byte aligned), fewer than 2^31 voxels (payload offsets are int
// words), at most 2^20 scan blocks
bool geom_ok(const df_volume &v)
{
    if (v.dims[0] <= 0 || v.dims[1] <= 0 || v.dims[2] <= 0 || v.dims[0] % 32 != 0) return false;
    if ((double)v.dims[0] * v.dims[1] * v.dims[2] >= 2147483648.0) return false;
    if (((uintptr_t)v.data & 15u) != 0) return false;
    return scan_fits(geom_of(v).nblocks);
}

struct WsLayout { BlockScan scan; int *total, *bad; };
WsLayout ws_of(void *ws, const PackGeom &g)
{
    WsLayout w;
    w.scan = block_scan_at((int *)ws, g.nblocks);
    w.total = (int *)ws + block_scan_ints(g.nblocks);
    w.bad = w.total + 1;
    return w;
}

__device__ __forceinline__ int class_words(int c) { return c == 0 ? 0 : (c == 1 ? 1 : BRICK_WORDS); }

struct BrickCoord { int x0, y0, z0; };
__device__ __forceinline__ BrickCoord brick_coord(const PackGeom &g, int b)
{
    const int bx = b % g.nbx, t = b / g.nbx;
    BrickCoord c;
    c.x0 = bx * DF_BRICK; c.y0 = (t % g.nby) * DF_BRICK; c.z0 = (t / g.nby) * DF_BRICK;
    return c;
}
// quad j of the brick: volume word index of its first voxel, or -1 when the row lies outside the volume (y or z past the edge)
__device__ __forceinline__ long long quad_index(const PackGeom &g, const BrickCoord &c, int j)
{
    const int r = j >> 1, y = c.y0 + (r & 7), z = c.z0 + (r >> 3);
    if (y >= g.Dy || z >= g.Dz) return -1;
    return ((long long)z * g.Dy + y) * g.Dx + c.x0 + (j & 1) * 4;
}

// exclusive payload offset (words) of the calling warp's brick: block prefix from the scan + the bricks of the earlier warps of the block
__device__ __forceinline__ int brick_offset(const PackGeom &g, const unsigned char *classes, const BlockScan &scan, int warp)
{
    int off = scan.base(blockIdx.x);
    for (int w = 0; w < warp; ++w) off += class_words(classes[blockIdx.x * PK_WARPS + w]);
    return off;
}

// classify: one class byte per brick, payload words per block.  The only full read of the volume (4 * V bytes).
__global__ void __launch_bounds__(PK_THREADS) pack_count_kernel(const uint32_t *__restrict__ vol, const PackGeom g, unsigned char *classes,
                                                                 int *block_counts)
{
    __shared__ int wwords[PK_WARPS];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int b = blockIdx.x * PK_WARPS + warp;
    int words = 0;
    if (b < g.nbricks) {                                              // uniform per warp
        const BrickCoord c = brick_coord(g, b);
        uint4 q[4];
        bool in[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const long long a = quad_index(g, c, lane + 32 * i);
            in[i] = a >= 0;
            q[i] = in[i] ? __ldg(reinterpret_cast<const uint4 *>(vol + a)) : make_uint4(0u, 0u, 0u, 0u);
        }
        const uint32_t w0 = __shfl_sync(0xffffffffu, q[0].x, 0);      // voxel (x0, y0, z0): always inside the volume
        bool same = true;
#pragma unroll
        for (int i = 0; i < 4; ++i)
            if (in[i]) same = same && q[i].x == w0 && q[i].y == w0 && q[i].z == w0 && q[i].w == w0;
        same = __all_sync(0xffffffffu, same);
        const int cls = same ? (w0 != 0u ? 1 : 0) : 2;
        if (lane == 0) classes[b] = (unsigned char)cls;
        words = class_words(cls);
    }
    if (lane == 0) wwords[warp] = words;
    __syncthreads();
    if (threadIdx.x == 0) {
        int s = 0;
#pragma unroll
        for (int w = 0; w < PK_WARPS; ++w) s += wwords[w];
        block_counts[blockIdx.x] = s;
    }
}

// emit: the payload in brick order; only the mixed bricks are read again.  Never writes at or past cap_words.
__global__ void __launch_bounds__(PK_THREADS) pack_emit_kernel(const uint32_t *__restrict__ vol, const PackGeom g, const unsigned char *classes,
                                                                const BlockScan scan, uint32_t *payload, size_t cap_words)
{
    __shared__ __align__(16) uint32_t stage[PK_WARPS][BRICK_WORDS];
    if (scan.counts[blockIdx.x] == 0) return;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int b = blockIdx.x * PK_WARPS + warp;
    if (b >= g.nbricks) return;
    const int cls = classes[b];
    if (cls == 0) return;
    const size_t off = (size_t)brick_offset(g, classes, scan, warp);
    const BrickCoord c = brick_coord(g, b);
    if (cls == 1) {
        if (lane == 0 && off < cap_words) payload[off] = vol[((size_t)c.z0 * g.Dy + c.y0) * g.Dx + c.x0];
        return;
    }
    uint4 q[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const long long a = quad_index(g, c, lane + 32 * i);
        q[i] = a >= 0 ? __ldg(reinterpret_cast<const uint4 *>(vol + a)) : make_uint4(0u, 0u, 0u, 0u);
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) reinterpret_cast<uint4 *>(stage[warp])[lane + 32 * i] = q[i];
    __syncwarp();
#pragma unroll
    for (int k = 0; k < BRICK_WORDS / 32; ++k) {                     // the brick's words start anywhere: coalesced scalar stores
        const size_t o = off + (size_t)(k * 32 + lane);
        if (o < cap_words) payload[o] = stage[warp][k * 32 + lane];
    }
}

// unpack, step 1: payload words per block from the class bytes; any byte outside {0, 1, 2} raises *bad
__global__ void __launch_bounds__(256) unpack_count_kernel(const unsigned char *classes, const PackGeom g, int *block_counts, int *bad)
{
    const int blk = blockIdx.x * blockDim.x + threadIdx.x;
    if (blk >= g.nblocks) return;
    int s = 0, wrong = 0;
    for (int w = 0; w < PK_WARPS; ++w) {
        const int b = blk * PK_WARPS + w;
        if (b >= g.nbricks) break;
        const int c = classes[b];
        if (c > 2) wrong = 1;
        else s += class_words(c);
    }
    block_counts[blk] = s;
    if (wrong) atomicOr(bad, 1);
}

// after the scan: total payload words (pack: -> bytes_out) or the validity of an unpack (-> status); one thread
__global__ void pack_finish_kernel(const int *total_words, const int *bad, unsigned long long expect_bytes, unsigned long long *bytes_out,
                                   int *status)
{
    const unsigned long long bytes = 4ull * (unsigned long long)*total_words;
    if (bytes_out) *bytes_out = bytes;
    if (status) *status = *bad ? DF_UNPACK_BAD_CLASS : (bytes != expect_bytes ? DF_UNPACK_BAD_LENGTH : 0);
}

// unpack, step 2: every voxel of the volume, brick by brick; nothing at all unless the checks passed (*status == 0)
__global__ void __launch_bounds__(PK_THREADS) unpack_write_kernel(uint32_t *__restrict__ vol, const PackGeom g, const unsigned char *classes,
                                                                   const BlockScan scan, const uint32_t *__restrict__ payload, const int *status)
{
    __shared__ __align__(16) uint32_t stage[PK_WARPS][BRICK_WORDS];
    if (*status != 0) return;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int b = blockIdx.x * PK_WARPS + warp;
    if (b >= g.nbricks) return;
    const int cls = classes[b];
    const BrickCoord c = brick_coord(g, b);
    const size_t off = (size_t)brick_offset(g, classes, scan, warp);
    if (cls == 2) {
#pragma unroll
        for (int k = 0; k < BRICK_WORDS / 32; ++k) stage[warp][k * 32 + lane] = __ldg(payload + off + k * 32 + lane);
        __syncwarp();
    }
    const uint32_t fill = cls == 1 ? __ldg(payload + off) : 0u;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int j = lane + 32 * i;
        const long long a = quad_index(g, c, j);
        if (a < 0) continue;
        const uint4 q = cls == 2 ? reinterpret_cast<const uint4 *>(stage[warp])[j] : make_uint4(fill, fill, fill, fill);
        *reinterpret_cast<uint4 *>(vol + a) = q;
    }
}

}  // namespace

extern "C" size_t df_volume_brick_count(df_volume vol) { return (size_t)geom_of(vol).nbricks; }

extern "C" size_t df_volume_pack_workspace_bytes(df_volume vol)
{
    return (block_scan_ints(geom_of(vol).nblocks) + 64) * sizeof(int);
}

extern "C" int df_volume_pack_count(df_volume vol, void *workspace, unsigned char *classes, unsigned long long *payload_bytes, void *stream)
{
    if (!geom_ok(vol) || !workspace || !classes || !payload_bytes) return (int)cudaErrorInvalidValue;
    const PackGeom g = geom_of(vol);
    const WsLayout w = ws_of(workspace, g);
    cudaStream_t s = (cudaStream_t)stream;
    pack_count_kernel<<<g.nblocks, PK_THREADS, 0, s>>>(vol.data, g, classes, w.scan.counts);
    DF_LAUNCH_CHECK();
    if (int st = scan_block_counts(w.scan, g.nblocks, 0x7fffffff, w.total, s)) return st;
    pack_finish_kernel<<<1, 1, 0, s>>>(w.total, nullptr, 0ull, payload_bytes, nullptr);
    DF_LAUNCH_CHECK();
    return 0;
}

extern "C" int df_volume_pack_emit(df_volume vol, const void *workspace, const unsigned char *classes, uint32_t *payload, size_t capacity, void *stream)
{
    if (!geom_ok(vol) || !workspace || !classes || (!payload && capacity)) return (int)cudaErrorInvalidValue;
    const PackGeom g = geom_of(vol);
    const WsLayout w = ws_of(const_cast<void *>(workspace), g);
    pack_emit_kernel<<<g.nblocks, PK_THREADS, 0, (cudaStream_t)stream>>>(vol.data, g, classes, w.scan, payload, capacity / 4);
    DF_LAUNCH_CHECK();
    return 0;
}

extern "C" int df_volume_unpack(df_volume vol, const unsigned char *classes, const uint32_t *payload, size_t payload_bytes, void *workspace,
                                int *status, void *stream)
{
    if (!geom_ok(vol) || !workspace || !classes || !status || (!payload && payload_bytes) || ((uintptr_t)payload & 3u)) return (int)cudaErrorInvalidValue;
    const PackGeom g = geom_of(vol);
    const WsLayout w = ws_of(workspace, g);
    cudaStream_t s = (cudaStream_t)stream;
    if (cudaMemsetAsync(w.bad, 0, sizeof(int), s) != cudaSuccess) return (int)cudaGetLastError();
    unpack_count_kernel<<<div_up(g.nblocks, 256), 256, 0, s>>>(classes, g, w.scan.counts, w.bad);
    DF_LAUNCH_CHECK();
    if (int st = scan_block_counts(w.scan, g.nblocks, 0x7fffffff, w.total, s)) return st;
    pack_finish_kernel<<<1, 1, 0, s>>>(w.total, w.bad, (unsigned long long)payload_bytes, nullptr, status);
    DF_LAUNCH_CHECK();
    unpack_write_kernel<<<g.nblocks, PK_THREADS, 0, s>>>(vol.data, g, classes, w.scan, payload, status);
    DF_LAUNCH_CHECK();
    return 0;
}
