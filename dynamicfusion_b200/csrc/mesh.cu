// mesh.cu -- triangle mesh over the extracted cloud (df_mesh_*, dfusion.h), sm_90a.
//
// The vertices are the cloud's points (extract.cu), so a triangle is three cloud indices.  The cloud emits its points in ascending
// (z, y, x) voxel order, +x, +y, +z within a voxel, over the volume walk of volscan.cuh, and every pass here walks the volume the same way
// and decides the points by the same crossing rule (crossing_axes).  The cloud index of the point a voxel emits on one axis is then
//   base[quad of the voxel] + points of the earlier voxels of that quad + points of that voxel on the earlier axes,
// where base[q] is the index of quad q's first point: its block's base in the scan of the per-block point counts plus the exclusive scan
// of the per-quad counts inside the block.  Kernels:
//   mesh_count_kernel        per block: cloud points (the recount that validates the cloud) and triangles; one thread per quad of VX cubes
//                            anchored at the quad's voxels, rows loaded with 16-byte loads when VX = 4;
//   scan_block_counts x 2    (volscan.cu) -> points total, triangle offsets and count;
//   mesh_status_kernel       points total against the cloud's count;
//   mesh_vertex_base_kernel  base[q] for every quad of the blocks that hold points (the table is read only there);
//   mesh_emit_kernel         the triangles of the blocks that have any, at their scanned offsets.
// Every pass skips the quads quad_skipped names.
#include "volscan.cuh"
#include "../../include/df_mc_table.h"

using namespace dfb;

namespace {

constexpr signed char kTris[256][DF_MC_ROW] = DF_MC_TRIANGLES_INIT;
struct TriCounts { unsigned char n[256]; };
constexpr TriCounts make_tri_counts()
{
    TriCounts c{};
    for (int i = 0; i < 256; ++i) {
        int k = 0;
        while (k < DF_MC_ROW && kTris[i][k] >= 0) ++k;
        c.n[i] = (unsigned char)(k / 3);
    }
    return c;
}
__constant__ TriCounts c_tri_counts = make_tri_counts();
__constant__ signed char c_tris[256][DF_MC_ROW] = DF_MC_TRIANGLES_INIT;
__constant__ signed char c_owner[12][4] = DF_MC_EDGE_OWNER_INIT;

// a corner of a polygonised cube: active, and F < 0 or F > 0 (not +-0, not NaN)
__device__ __forceinline__ bool corner_ok(uint32_t v) { const float F = vox_f(v); return vox_active(v) && (F < 0.f || F > 0.f); }

// voxels x0 .. x0 + N - 1 of row (y, z), 0 (inactive) outside the volume; the first VX of them in one 16-byte load when VX = 4
template <int VX, int N>
__device__ __forceinline__ void load_row(const VolumeWalk &p, int x0, int y, int z, uint32_t (&r)[N])
{
#pragma unroll
    for (int j = 0; j < N; ++j) r[j] = 0u;
    if (y >= p.Dy || z >= p.Dz) return;
    const uint32_t *row = p.data + ((size_t)z * p.Dy + y) * p.Dx;
    if (VX == 4) {
        const uint4 q = __ldg(reinterpret_cast<const uint4 *>(row + x0));
        r[0] = q.x; r[1 % N] = q.y; r[2 % N] = q.z; r[3 % N] = q.w;
    } else {
        r[0] = __ldg(row + x0);
    }
#pragma unroll
    for (int j = VX; j < N; ++j)
        if (x0 + j < p.Dx) r[j] = __ldg(row + x0 + j);
}

// case of the cube anchored at (x0 + j, y, z) (dfusion.h: the rule; df_mc_table.h: corner numbering), -1 when it is not polygonised.
// A, B, C, D: rows (y, z), (y + 1, z), (y, z + 1), (y + 1, z + 1) from x0.
template <int N>
__device__ __forceinline__ int cube_case(const VolumeWalk &p, const uint32_t (&A)[N], const uint32_t (&B)[N], const uint32_t (&C)[N],
                                         const uint32_t (&D)[N], int j, int x0, int y, int z)
{
    if (x0 + j > p.Dx - 2 || y > p.Dy - 2 || z > p.Dz - 3) return -1;
    const uint32_t c[8] = {A[j], A[j + 1], B[j + 1], B[j], C[j], C[j + 1], D[j + 1], D[j]};
    int cs = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        if (!corner_ok(c[i])) return -1;
        if (vox_f(c[i]) < 0.f) cs |= 1 << i;
    }
    return cs;
}

// cloud points of the quad at v0 (rows A, B, C from x0, A with one voxel more)
template <int VX>
__device__ __forceinline__ int quad_points(const VolumeWalk &p, const QuadCoord &c, const uint32_t (&A)[VX + 1], const uint32_t (&B)[VX + 1],
                                           const uint32_t (&C)[VX + 1])
{
    int n = 0;
#pragma unroll
    for (int j = 0; j < VX; ++j) n += __popc(crossing_axes(p, A[j], A[j + 1], B[j], C[j], c.x0 + j, c.y, c.z));
    return n;
}

template <int VX>
__global__ void __launch_bounds__(WALK_THREADS) mesh_count_kernel(const VolumeWalk p, int *point_counts, int *tri_counts)
{
    __shared__ int sums[2][WALK_THREADS / 32];
    int np = 0, nt = 0;
#pragma unroll
    for (int i = 0; i < WALK_QPT; ++i) {
        const size_t v0 = quad_voxel<VX>(i);
        if (quad_skipped(p, v0)) continue;
        const QuadCoord c = quad_coord(p, v0);
        uint32_t A[VX + 1], B[VX + 1], C[VX + 1], D[VX + 1];
        load_row<VX>(p, c.x0, c.y, c.z, A);
        bool any = false;
#pragma unroll
        for (int j = 0; j < VX; ++j) any |= vox_active(A[j]);
        if (!any) continue;                                   // no point and no anchored cube
        load_row<VX>(p, c.x0, c.y + 1, c.z, B);
        load_row<VX>(p, c.x0, c.y, c.z + 1, C);
        load_row<VX>(p, c.x0, c.y + 1, c.z + 1, D);
        np += quad_points<VX>(p, c, A, B, C);
#pragma unroll
        for (int j = 0; j < VX; ++j) {
            const int cs = cube_case(p, A, B, C, D, j, c.x0, c.y, c.z);
            if (cs > 0 && cs < 255) nt += c_tri_counts.n[cs];
        }
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        np += __shfl_xor_sync(0xffffffffu, np, o);
        nt += __shfl_xor_sync(0xffffffffu, nt, o);
    }
    if (lane == 0) { sums[0][warp] = np; sums[1][warp] = nt; }
    __syncthreads();
    if (threadIdx.x == 0) {
        int a = 0, b = 0;
#pragma unroll
        for (int w = 0; w < WALK_THREADS / 32; ++w) { a += sums[0][w]; b += sums[1][w]; }
        point_counts[blockIdx.x] = a;
        tri_counts[blockIdx.x] = b;
    }
}

__global__ void mesh_status_kernel(const int *points_total, const int *cloud_count, int *status)
{
    *status = *points_total != *cloud_count ? DF_MESH_CLOUD_MISMATCH : 0;
}

template <int VX>
__global__ void __launch_bounds__(WALK_THREADS) mesh_vertex_base_kernel(const VolumeWalk p, const BlockScan points, int *base)
{
    if (points.counts[blockIdx.x] == 0) return;
    int run = points.base(blockIdx.x);
#pragma unroll
    for (int i = 0; i < WALK_QPT; ++i) {                              // quads in order i * WALK_THREADS + tid, as the cloud's points
        const size_t v0 = quad_voxel<VX>(i);
        int n = 0;
        if (!quad_skipped(p, v0)) {
            const QuadCoord c = quad_coord(p, v0);
            uint32_t A[VX + 1], B[VX + 1], C[VX + 1];
            load_row<VX>(p, c.x0, c.y, c.z, A);
            load_row<VX>(p, c.x0, c.y + 1, c.z, B);
            load_row<VX>(p, c.x0, c.y, c.z + 1, C);
            n = quad_points<VX>(p, c, A, B, C);
        }
        int total;
        const int excl = block_exclusive_scan<WALK_THREADS>(n, &total);
        if (v0 < p.nvox) base[v0 / VX] = run + excl;
        run += total;
    }
}

template <int VX>
__global__ void __launch_bounds__(WALK_THREADS) mesh_emit_kernel(const VolumeWalk p, const BlockScan tris, const int *base, int3 *out,
                                                               int capacity)
{
    if (tris.counts[blockIdx.x] == 0) return;
    int run = tris.base(blockIdx.x);
#pragma unroll 1
    for (int i = 0; i < WALK_QPT; ++i) {
        const size_t v0 = quad_voxel<VX>(i);
        QuadCoord c = {0, 0, 0};
        uint32_t A[VX + 2], B[VX + 2], C[VX + 2], D[VX + 2];
        int cs[VX];
        int n = 0;
#pragma unroll
        for (int j = 0; j < VX; ++j) cs[j] = -1;
        if (!quad_skipped(p, v0)) {
            c = quad_coord(p, v0);
            load_row<VX>(p, c.x0, c.y, c.z, A);
            load_row<VX>(p, c.x0, c.y + 1, c.z, B);
            load_row<VX>(p, c.x0, c.y, c.z + 1, C);
            load_row<VX>(p, c.x0, c.y + 1, c.z + 1, D);
#pragma unroll
            for (int j = 0; j < VX; ++j) {
                cs[j] = cube_case(p, A, B, C, D, j, c.x0, c.y, c.z);
                if (cs[j] > 0 && cs[j] < 255) n += c_tri_counts.n[cs[j]];
            }
        }
        int total;
        int k = run + block_exclusive_scan<WALK_THREADS>(n, &total);
        run += total;
        if (n == 0) continue;
        // the voxels that own this quad's cube edges: rows A, B, C, D (r = dy + 2 dz), voxels x0 .. x0 + VX; their points need the rows
        // one further in y or z
        uint32_t E[VX + 1], F[VX + 1], G[VX + 1], H[VX + 1];
        load_row<VX>(p, c.x0, c.y + 2, c.z, E);
        load_row<VX>(p, c.x0, c.y, c.z + 2, F);
        load_row<VX>(p, c.x0, c.y + 2, c.z + 1, G);
        load_row<VX>(p, c.x0, c.y + 1, c.z + 2, H);
        int fl[4][VX + 1], first[4][VX + 1];
#pragma unroll
        for (int j = 0; j <= VX; ++j) {
            const int x = c.x0 + j;
            fl[0][j] = crossing_axes(p, A[j], A[j + 1], B[j], C[j], x, c.y, c.z);
            fl[1][j] = crossing_axes(p, B[j], B[j + 1], E[j], D[j], x, c.y + 1, c.z);
            fl[2][j] = crossing_axes(p, C[j], C[j + 1], D[j], F[j], x, c.y, c.z + 1);
            fl[3][j] = crossing_axes(p, D[j], D[j + 1], G[j], H[j], x, c.y + 1, c.z + 1);
        }
        // cloud index of each owner's first point; voxel x0 + VX is the first of the next quad.  base[] is read only for quads with points.
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            const size_t q = (((size_t)(c.z + (r >> 1)) * p.Dy + (c.y + (r & 1))) * p.Dx + c.x0) / VX;
            int any = 0;
#pragma unroll
            for (int j = 0; j < VX; ++j) any |= fl[r][j];
            int b = any ? base[q] : 0;
#pragma unroll
            for (int j = 0; j < VX; ++j) { first[r][j] = b; b += __popc(fl[r][j]); }
            first[r][VX] = fl[r][VX] ? base[q + 1] : 0;
        }
#pragma unroll
        for (int j = 0; j < VX; ++j) {
            const int cj = cs[j];
            if (cj <= 0 || cj >= 255) continue;
            const int nt = c_tri_counts.n[cj];
            for (int t = 0; t < nt; ++t) {
                int idx[3];
#pragma unroll
                for (int m = 0; m < 3; ++m) {
                    const int e = c_tris[cj][3 * t + m];
                    const int r = c_owner[e][1] + 2 * c_owner[e][2], jj = j + c_owner[e][0], axis = c_owner[e][3];
                    idx[m] = first[r][jj] + __popc(fl[r][jj] & ((1 << axis) - 1));
                }
                if (k < capacity) out[k] = make_int3(idx[0], idx[1], idx[2]);
                ++k;
            }
        }
    }
}

bool params_ok(const df_volume &vol)
{
    if (!vol.data || vol.dims[0] <= 0 || vol.dims[1] <= 0 || vol.dims[2] <= 0) return false;
    return scan_fits(volume_walk(vol, nullptr).nblocks);
}

// the scans of the point and triangle counts, the points total (+ 64 ints), then base[] (one int per quad)
struct WsLayout { BlockScan points, tris; int *points_total, *base; };
WsLayout ws_of(void *ws, const VolumeWalk &p)
{
    WsLayout w;
    int *q = (int *)ws;
    w.points = block_scan_at(q, p.nblocks);
    w.tris = block_scan_at(q += block_scan_ints(p.nblocks), p.nblocks);
    w.points_total = q + block_scan_ints(p.nblocks);
    w.base = w.points_total + 64;
    return w;
}

}  // namespace

extern "C" size_t df_mesh_workspace_bytes(df_volume vol)
{
    const VolumeWalk p = volume_walk(vol, nullptr);
    const size_t nquads = (p.nvox + p.vx - 1) / p.vx;
    return (2 * block_scan_ints(p.nblocks) + 64 + nquads) * sizeof(int);
}

extern "C" int df_mesh_count(df_volume vol, const unsigned char *activity, const int *cloud_count_dev, void *workspace, int *tri_count_dev,
                             int *status_dev, void *stream)
{
    if (!params_ok(vol) || !cloud_count_dev || !workspace || !tri_count_dev || !status_dev) return (int)cudaErrorInvalidValue;
    const VolumeWalk p = volume_walk(vol, activity);
    const WsLayout w = ws_of(workspace, p);
    cudaStream_t s = (cudaStream_t)stream;
    if (p.vx == 4) mesh_count_kernel<4><<<p.nblocks, WALK_THREADS, 0, s>>>(p, w.points.counts, w.tris.counts);
    else mesh_count_kernel<1><<<p.nblocks, WALK_THREADS, 0, s>>>(p, w.points.counts, w.tris.counts);
    DF_LAUNCH_CHECK();
    if (int st = scan_block_counts(w.points, p.nblocks, 0x7fffffff, w.points_total, s)) return st;
    if (int st = scan_block_counts(w.tris, p.nblocks, 0x7fffffff, tri_count_dev, s)) return st;
    mesh_status_kernel<<<1, 1, 0, s>>>(w.points_total, cloud_count_dev, status_dev);
    DF_LAUNCH_CHECK();
    if (p.vx == 4) mesh_vertex_base_kernel<4><<<p.nblocks, WALK_THREADS, 0, s>>>(p, w.points, w.base);
    else mesh_vertex_base_kernel<1><<<p.nblocks, WALK_THREADS, 0, s>>>(p, w.points, w.base);
    DF_LAUNCH_CHECK();
    return 0;
}

extern "C" int df_mesh_emit(df_volume vol, const unsigned char *activity, const void *workspace, int32_t *tris, int capacity, void *stream)
{
    if (!params_ok(vol) || !workspace || (!tris && capacity > 0)) return (int)cudaErrorInvalidValue;
    const VolumeWalk p = volume_walk(vol, activity);
    const WsLayout w = ws_of(const_cast<void *>(workspace), p);
    cudaStream_t s = (cudaStream_t)stream;
    if (p.vx == 4) mesh_emit_kernel<4><<<p.nblocks, WALK_THREADS, 0, s>>>(p, w.tris, w.base, (int3 *)tris, capacity);
    else mesh_emit_kernel<1><<<p.nblocks, WALK_THREADS, 0, s>>>(p, w.tris, w.base, (int3 *)tris, capacity);
    DF_LAUNCH_CHECK();
    return 0;
}
