// warp_common.cuh -- device-side warp-field primitives shared by warp.cu and solve.cu:
// exact 8-NN over a GPU-resident node table, node weights, dual-quaternion blend.
// Replaces the CPU path of the reference: nanoflann kd-tree queries (kfusion/src/warp_field.cpp:247-251,
// kfusion/include/nanoflann/nanoflann.hpp:901-915) and the scalar DQB loop (warp_field.cpp:180-241).
#pragma once
#include "df_common.cuh"

namespace dfb {

constexpr int KNN_TILE = 1024;       // nodes staged per shared-memory tile (SoA, 12 KB)

struct KnnSmem { float x[KNN_TILE], y[KNN_TILE], z[KNN_TILE]; };

// Exact 8 nearest nodes of q by exhaustive scan in ascending node index.  Result-set semantics of nanoflann's
// KNNResultSet::addPoint (nanoflann.hpp:110-131): accept iff dist < current worst (strict), equal distances keep
// visiting order (=> ties resolve to the lower node index); distance d0*d0 + d1*d1 + d2*d2 evaluated left to right in
// float (knn_point_cloud.hpp:26-32).  ALL threads of the block must call this (tile staging uses __syncthreads);
// `valid` = false skips the scan for this thread (NaN query).
__device__ __forceinline__ void knn8_scan(const float *__restrict__ nodes, int M, bool valid, float qx, float qy, float qz,
                                          KnnSmem &sm, int (&bi)[8], float (&bd)[8])
{
#pragma unroll
    for (int i = 0; i < 8; ++i) { bi[i] = -1; bd[i] = 3.402823466e+38f; }
    const int tid = threadIdx.x + threadIdx.y * blockDim.x;
    const int nthreads = blockDim.x * blockDim.y;
    for (int base = 0; base < M; base += KNN_TILE) {
        const int n = min(KNN_TILE, M - base);
        __syncthreads();
        for (int i = tid; i < n; i += nthreads) {
            const float *v = nodes + (size_t)(base + i) * DF_NODE_STRIDE;
            sm.x[i] = __ldg(v); sm.y[i] = __ldg(v + 1); sm.z[i] = __ldg(v + 2);
        }
        __syncthreads();
        if (!valid) continue;
#pragma unroll 4
        for (int i = 0; i < n; ++i) {
            const float d0 = qx - sm.x[i], d1 = qy - sm.y[i], d2 = qz - sm.z[i];
            const float dist = d0 * d0 + d1 * d1 + d2 * d2;
            if (dist < bd[7]) {
                bd[7] = dist; bi[7] = base + i;
#pragma unroll
                for (int k = 7; k > 0; --k) {
                    if (bd[k] < bd[k - 1]) {
                        const float td = bd[k]; bd[k] = bd[k - 1]; bd[k - 1] = td;
                        const int ti = bi[k]; bi[k] = bi[k - 1]; bi[k - 1] = ti;
                    }
                }
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------------------------
// Uniform node grid: the GPU-resident replacement of the reference's nanoflann kd-tree (warp_field.cpp:17-27,275-282).
// Node vertices never move after WarpField::init, so the grid is built once (nodegrid.cu) and every query walks cubic
// shells of cells around its own cell until the 8 best cannot be beaten any more.  Candidates are ranked by
// (squared distance, node index), so the result is exactly the exhaustive scan's (knn8_scan) whatever the visiting order.
constexpr int NODEGRID_MAX_RES = 64;
constexpr int NODEGRID_ORDER_MAX_M = 8192;
constexpr int NODEGRID_BVH_LEAF = 8;

struct NodeGridHeader {
    float ox, oy, oz, cell, inv_cell;
    int gx, gy, gz, M, ncell;
    int pad[6];            // pad[0], pad[1]: byte offsets of the Morton order[] / slot[] arrays; pad[2], pad[3], pad[4]: BVH boxes, BVH
                           // leaves (byte offsets) and leaf count L (0 = absent)
};   // 64 bytes, followed by: int cell_start[ncell + 1] (padded to 16 B), float4 sorted[M] = (x, y, z, index bits)

__device__ __forceinline__ const int *nodegrid_cell_start(const void *grid) { return reinterpret_cast<const int *>(reinterpret_cast<const char *>(grid) + 64); }
__device__ __forceinline__ const float4 *nodegrid_sorted(const void *grid, int ncell)
{ return reinterpret_cast<const float4 *>(reinterpret_cast<const char *>(grid) + 64 + (((size_t)(ncell + 1) * 4 + 15) & ~(size_t)15)); }

// Morton ordering of the nodes (nodegrid.cu step 5): order[rank] = node index, slot[node] = rank; nullptr when absent
__device__ __forceinline__ const int *nodegrid_order(const void *grid)
{ const int o = reinterpret_cast<const NodeGridHeader *>(grid)->pad[0]; return o ? reinterpret_cast<const int *>(reinterpret_cast<const char *>(grid) + o) : nullptr; }
__device__ __forceinline__ const int *nodegrid_slot(const void *grid)
{ const int o = reinterpret_cast<const NodeGridHeader *>(grid)->pad[1]; return o ? reinterpret_cast<const int *>(reinterpret_cast<const char *>(grid) + o) : nullptr; }

__device__ __forceinline__ void knn8_insert_lex(int (&bi)[8], float (&bd)[8], float dist, int idx)
{
    if (dist < bd[7] || (dist == bd[7] && idx < bi[7])) {
        bd[7] = dist; bi[7] = idx;
#pragma unroll
        for (int k = 7; k > 0; --k) {
            if (bd[k] < bd[k - 1] || (bd[k] == bd[k - 1] && bi[k] < bi[k - 1])) {
                const float td = bd[k]; bd[k] = bd[k - 1]; bd[k - 1] = td;
                const int ti = bi[k]; bi[k] = bi[k - 1]; bi[k - 1] = ti;
            }
        }
    }
}

// Shell walks are cheap while the query is within a cell or two of the nodes; a query far outside the node cloud (the reference
// feeds camera-frame points to a world-frame field, kinfu.cpp:356-361, so this is the common case once the camera has moved)
// would visit thousands of empty cells.  Such a query is answered by a bounding-volume hierarchy instead (nodegrid.cu step 6):
// depth-first, nearer child first, a subtree is skipped when the squared distance to its box exceeds the current 8th best.
// The box distance is formed with the same float operations as a node distance ((dx*dx + dy*dy) + dz*dz, |dx| no larger than
// for any node inside), so it never exceeds the distance computed for a node of that subtree: pruning is exact, and since all
// paths rank by (distance, index) the result does not depend on which one ran.  Without a BVH the fallback is exhaustive.
constexpr int KNN_SHELL_CAP = 1;

__device__ __forceinline__ float bvh_box_dist2(const float4 lo, const float4 hi, float qx, float qy, float qz)
{
    const float d0 = fmaxf(fmaxf(lo.x - qx, qx - hi.x), 0.f), d1 = fmaxf(fmaxf(lo.y - qy, qy - hi.y), 0.f), d2 = fmaxf(fmaxf(lo.z - qz, qz - hi.z), 0.f);
    return d0 * d0 + d1 * d1 + d2 * d2;
}

__device__ __forceinline__ void knn8_bvh(const float4 *__restrict__ box, const float4 *__restrict__ leaf, int L, float qx, float qy, float qz,
                                         int (&bi)[8], float (&bd)[8])
{
    int stack_i[24];
    float stack_d[24];
    int sp = 0;
    stack_i[sp] = 0; stack_d[sp] = 0.f; ++sp;
    while (sp > 0) {
        --sp;
        const int i = stack_i[sp];
        if (stack_d[sp] > bd[7]) continue;                       // strict: an equal distance may still win on the index
        if (i >= L - 1) {
            const float4 *e = leaf + (size_t)(i - (L - 1)) * NODEGRID_BVH_LEAF;
#pragma unroll
            for (int k = 0; k < NODEGRID_BVH_LEAF; ++k) {
                const float4 nd = __ldg(e + k);
                const float d0 = qx - nd.x, d1 = qy - nd.y, d2 = qz - nd.z;
                knn8_insert_lex(bi, bd, d0 * d0 + d1 * d1 + d2 * d2, __float_as_int(nd.w));   // padding: distance inf, index INT_MAX
            }
        } else {
            const int a = 2 * i + 1, b = a + 1;
            const float da = bvh_box_dist2(__ldg(box + 2 * a), __ldg(box + 2 * a + 1), qx, qy, qz);
            const float db = bvh_box_dist2(__ldg(box + 2 * b), __ldg(box + 2 * b + 1), qx, qy, qz);
            const bool a_first = da <= db;
            const int far_i = a_first ? b : a, near_i = a_first ? a : b;
            const float far_d = a_first ? db : da, near_d = a_first ? da : db;
            if (far_d <= bd[7]) { stack_i[sp] = far_i; stack_d[sp] = far_d; ++sp; }      // empty subtrees have distance inf (NaN-free: inf - q)
            if (near_d <= bd[7]) { stack_i[sp] = near_i; stack_d[sp] = near_d; ++sp; }
        }
    }
}

// knn8_bvh with a caller-supplied upper bound on the 8th-nearest distance (e.g. the largest distance from the query to ANY eight
// distinct nodes, such as the neighbours of an adjacent query): the set starts empty, candidates farther than `limit` are dropped
// before the insertion and subtrees farther than min(limit, current 8th best) are not entered.  The true eight nearest all lie
// within `limit` (distances are formed by the same float operations everywhere, so a node that defined the bound is found again
// with exactly that distance) and ranking is by (distance, index): the result equals knn8_bvh's / the exhaustive scan's.
__device__ __forceinline__ void knn8_bvh_bounded(const float4 *__restrict__ box, const float4 *__restrict__ leaf, int L, float qx, float qy, float qz,
                                                 float limit, int (&bi)[8], float (&bd)[8])
{
#pragma unroll
    for (int i = 0; i < 8; ++i) { bi[i] = 0x7fffffff; bd[i] = 3.402823466e+38f; }
    int stack_i[24];
    float stack_d[24];
    int sp = 0;
    stack_i[sp] = 0; stack_d[sp] = 0.f; ++sp;
    while (sp > 0) {
        --sp;
        const int i = stack_i[sp];
        const float cut = fminf(bd[7], limit);
        if (stack_d[sp] > cut) continue;
        if (i >= L - 1) {
            const float4 *e = leaf + (size_t)(i - (L - 1)) * NODEGRID_BVH_LEAF;
#pragma unroll
            for (int k = 0; k < NODEGRID_BVH_LEAF; ++k) {
                const float4 nd = __ldg(e + k);
                const float d0 = qx - nd.x, d1 = qy - nd.y, d2 = qz - nd.z;
                const float dist = d0 * d0 + d1 * d1 + d2 * d2;
                if (dist <= limit) knn8_insert_lex(bi, bd, dist, __float_as_int(nd.w));       // padding has distance inf
            }
        } else {
            const int a = 2 * i + 1, b = a + 1;
            const float da = bvh_box_dist2(__ldg(box + 2 * a), __ldg(box + 2 * a + 1), qx, qy, qz);
            const float db = bvh_box_dist2(__ldg(box + 2 * b), __ldg(box + 2 * b + 1), qx, qy, qz);
            const bool a_first = da <= db;
            const int far_i = a_first ? b : a, near_i = a_first ? a : b;
            const float far_d = a_first ? db : da, near_d = a_first ? da : db;
            if (far_d <= cut) { stack_i[sp] = far_i; stack_d[sp] = far_d; ++sp; }
            if (near_d <= cut) { stack_i[sp] = near_i; stack_d[sp] = near_d; ++sp; }
        }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) if (bi[i] == 0x7fffffff) bi[i] = -1;
}

// knn8_bvh started from eight KNOWN nodes instead of an empty set: on entry bi[] holds eight distinct valid node indices and bd[] their
// squared distances to the query, in any order (e.g. the neighbours of an adjacent query).  They are sorted by (distance, index) with a
// 19-comparator network and the branch-and-bound then runs with the 8th of them as its bound from the first box on; a candidate that would
// enter the set is first checked against the eight indices held (a seed node met again in its leaf).  Same result as knn8_bvh: the final
// set is the (distance, index)-smallest eight of all nodes.  A profile of the first version of the warped-fusion kernel (search from an
// empty set with a distance limit): a quarter of all instructions were insertions -- far from the node cloud ~30 nodes are nearly equidistant and each
// query re-inserted ~18 of them -- with half of the lanes active.
__device__ __forceinline__ void knn8_cswap_lex(float &da, int &ia, float &db, int &ib)
{
    if (db < da || (db == da && ib < ia)) { const float td = da; da = db; db = td; const int ti = ia; ia = ib; ib = ti; }
}

__device__ __forceinline__ void knn8_bvh_seeded(const float4 *__restrict__ box, const float4 *__restrict__ leaf, int L, float qx, float qy, float qz,
                                                int (&bi)[8], float (&bd)[8])
{
#define DF_CS(a, b) knn8_cswap_lex(bd[a], bi[a], bd[b], bi[b])
    DF_CS(0, 1); DF_CS(2, 3); DF_CS(4, 5); DF_CS(6, 7);
    DF_CS(0, 2); DF_CS(1, 3); DF_CS(4, 6); DF_CS(5, 7);
    DF_CS(1, 2); DF_CS(5, 6);
    DF_CS(0, 4); DF_CS(1, 5); DF_CS(2, 6); DF_CS(3, 7);
    DF_CS(2, 4); DF_CS(3, 5);
    DF_CS(1, 2); DF_CS(3, 4); DF_CS(5, 6);
#undef DF_CS
    int stack_i[24];
    float stack_d[24];
    int sp = 0;
    stack_i[sp] = 0; stack_d[sp] = 0.f; ++sp;
    while (sp > 0) {
        --sp;
        const int i = stack_i[sp];
        if (stack_d[sp] > bd[7]) continue;                       // strict: an equal distance may still win on the index
        if (i >= L - 1) {
            const float4 *e = leaf + (size_t)(i - (L - 1)) * NODEGRID_BVH_LEAF;
#pragma unroll
            for (int k = 0; k < NODEGRID_BVH_LEAF; ++k) {
                const float4 nd = __ldg(e + k);
                const float d0 = qx - nd.x, d1 = qy - nd.y, d2 = qz - nd.z;
                const float dist = d0 * d0 + d1 * d1 + d2 * d2;
                const int idx = __float_as_int(nd.w);
                if (dist < bd[7] || (dist == bd[7] && idx < bi[7])) {
                    const bool held = idx == bi[0] || idx == bi[1] || idx == bi[2] || idx == bi[3] || idx == bi[4] || idx == bi[5] || idx == bi[6];
                    if (!held) knn8_insert_lex(bi, bd, dist, idx);
                }
            }
        } else {
            const int a = 2 * i + 1, b = a + 1;
            const float da = bvh_box_dist2(__ldg(box + 2 * a), __ldg(box + 2 * a + 1), qx, qy, qz);
            const float db = bvh_box_dist2(__ldg(box + 2 * b), __ldg(box + 2 * b + 1), qx, qy, qz);
            const bool a_first = da <= db;
            const int far_i = a_first ? b : a, near_i = a_first ? a : b;
            const float far_d = a_first ? db : da, near_d = a_first ? da : db;
            if (far_d <= bd[7]) { stack_i[sp] = far_i; stack_d[sp] = far_d; ++sp; }
            if (near_d <= bd[7]) { stack_i[sp] = near_i; stack_d[sp] = near_d; ++sp; }
        }
    }
}

// The eight entries of the leaf a greedy descent reaches (nearer child at every level, no backtracking), with their squared distances:
// a seed for knn8_bvh_seeded when no neighbouring result is at hand.  false when that leaf is padded (fewer than eight nodes).
__device__ __forceinline__ bool knn8_bvh_greedy_seed(const float4 *__restrict__ box, const float4 *__restrict__ leaf, int L, float qx, float qy, float qz,
                                                     int (&bi)[8], float (&bd)[8])
{
    int i = 0;
    while (i < L - 1) {
        const int a = 2 * i + 1, b = a + 1;
        const float da = bvh_box_dist2(__ldg(box + 2 * a), __ldg(box + 2 * a + 1), qx, qy, qz);
        const float db = bvh_box_dist2(__ldg(box + 2 * b), __ldg(box + 2 * b + 1), qx, qy, qz);
        i = da <= db ? a : b;
    }
    const float4 *e = leaf + (size_t)(i - (L - 1)) * NODEGRID_BVH_LEAF;
    bool full = true;
#pragma unroll
    for (int k = 0; k < NODEGRID_BVH_LEAF; ++k) {
        const float4 nd = __ldg(e + k);
        const float d0 = qx - nd.x, d1 = qy - nd.y, d2 = qz - nd.z;
        bd[k] = d0 * d0 + d1 * d1 + d2 * d2;
        bi[k] = __float_as_int(nd.w);
        full = full && bd[k] < 3.402823466e+38f;                 // padding: distance inf, index INT_MAX
    }
    return full;
}

__device__ __forceinline__ void knn8_grid(const void *__restrict__ grid, bool valid, float qx, float qy, float qz, int (&bi)[8], float (&bd)[8])
{
#pragma unroll
    for (int i = 0; i < 8; ++i) { bi[i] = 0x7fffffff; bd[i] = 3.402823466e+38f; }
    if (valid) {
        const NodeGridHeader h = *reinterpret_cast<const NodeGridHeader *>(grid);
        const int *cell_start = nodegrid_cell_start(grid);
        const float4 *sorted = nodegrid_sorted(grid, h.ncell);
        const int cx = min(max((int)floorf((qx - h.ox) * h.inv_cell), 0), h.gx - 1);
        const int cy = min(max((int)floorf((qy - h.oy) * h.inv_cell), 0), h.gy - 1);
        const int cz = min(max((int)floorf((qz - h.oz) * h.inv_cell), 0), h.gz - 1);
        const int rmax = max(max(h.gx, h.gy), h.gz);
        bool done = false;
        for (int r = 0; r <= rmax; ++r) {
            // shells 0..r-1 are done: every unvisited node sits in a cell at Chebyshev distance >= r from (cx,cy,cz), i.e. at
            // least (r-1)*cell away from the query (the query lies anywhere inside its own, possibly clamped, cell)
            if (r >= 2 && bi[7] != 0x7fffffff) {
                const float bound = (float)(r - 1) * h.cell * 0.999f;
                if (bound * bound > bd[7]) { done = true; break; }
            }
            if (r > KNN_SHELL_CAP) break;
            // Cells of one grid row (fixed y, z) are consecutive in memory, and so are their nodes: a row that lies on the shell
            // (|dz| == r or |dy| == r) is ONE contiguous run of nodes for the whole x-range, an interior row contributes only its two
            // end cells.  Rows whose box is farther than the current 8th best (FLT_MAX until eight candidates are known) are skipped;
            // the box is widened by 1e-4 cell and the bound taken 0.01 % low, so no node is lost to rounding.
            const float slack = h.cell * 1e-4f;
            for (int z = cz - r; z <= cz + r; ++z) {
                if (z < 0 || z >= h.gz) continue;
                const float zlo = h.oz + (float)z * h.cell - slack, zhi = zlo + h.cell + 2.f * slack;
                const float ez = fmaxf(fmaxf(zlo - qz, qz - zhi), 0.f);
                if (ez * ez * 0.9999f > bd[7]) continue;
                for (int y = cy - r; y <= cy + r; ++y) {
                    if (y < 0 || y >= h.gy) continue;
                    const float ylo = h.oy + (float)y * h.cell - slack, yhi = ylo + h.cell + 2.f * slack;
                    const float ey = fmaxf(fmaxf(ylo - qy, qy - yhi), 0.f);
                    if ((ez * ez + ey * ey) * 0.9999f > bd[7]) continue;
                    const bool shell = (z == cz - r) || (z == cz + r) || (y == cy - r) || (y == cy + r);
                    const int row = h.gx * (y + h.gy * z);
                    const int x0 = max(cx - r, 0), x1 = min(cx + r, h.gx - 1);
                    // segment 0: the whole x-range (shell row) or the left end cell; segment 1: the right end cell of an interior row
                    for (int seg = 0; seg < (shell || r == 0 ? 1 : 2); ++seg) {
                        int xa, xb;
                        if (shell || r == 0) { xa = x0; xb = x1; }
                        else if (seg == 0) { xa = xb = cx - r; }
                        else { xa = xb = cx + r; }
                        if (xa < 0 || xb >= h.gx || xa > xb) continue;
                        const int b = __ldg(cell_start + row + xa), e = __ldg(cell_start + row + xb + 1);
                        for (int it = b; it < e; ++it) {
                            const float4 nd = __ldg(sorted + it);
                            const float d0 = qx - nd.x, d1 = qy - nd.y, d2 = qz - nd.z;
                            knn8_insert_lex(bi, bd, d0 * d0 + d1 * d1 + d2 * d2, __float_as_int(nd.w));
                        }
                    }
                }
            }
            if (r == rmax) done = true;                       // every cell has been visited
        }
        if (!done) {
            if (h.pad[2]) {
                // Far query: branch-and-bound over the k-d BVH, SEEDED (round 2; the warped-fusion kernel showed what an unseeded search
                // costs far from the cloud: ~30 nearly equidistant nodes, 18 of them inserted and evicted again per query).  The seed is
                // the eight candidates the visited shells produced when there are eight, else the leaf a greedy descent reaches; either
                // is eight real nodes with their exact distances, so the result is the exhaustive scan's (knn8_bvh_seeded).
                const float4 *box = reinterpret_cast<const float4 *>(reinterpret_cast<const char *>(grid) + h.pad[2]);
                const float4 *leaf = reinterpret_cast<const float4 *>(reinterpret_cast<const char *>(grid) + h.pad[3]);
                bool seeded = bi[7] != 0x7fffffff;
                if (!seeded) seeded = knn8_bvh_greedy_seed(box, leaf, h.pad[4], qx, qy, qz, bi, bd);
                if (seeded) knn8_bvh_seeded(box, leaf, h.pad[4], qx, qy, qz, bi, bd);
                else {
#pragma unroll
                    for (int i = 0; i < 8; ++i) { bi[i] = 0x7fffffff; bd[i] = 3.402823466e+38f; }
                    knn8_bvh(box, leaf, h.pad[4], qx, qy, qz, bi, bd);
                }
            } else {
#pragma unroll
            for (int i = 0; i < 8; ++i) { bi[i] = 0x7fffffff; bd[i] = 3.402823466e+38f; }
#pragma unroll 4
            for (int it = 0; it < h.M; ++it) {
                const float4 nd = __ldg(sorted + it);
                const float d0 = qx - nd.x, d1 = qy - nd.y, d2 = qz - nd.z;
                knn8_insert_lex(bi, bd, d0 * d0 + d1 * d1 + d2 * d2, __float_as_int(nd.w));
            }
            }
        }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) if (bi[i] == 0x7fffffff) bi[i] = -1;
}

// Vertex handled by thread `tid` of 256-thread block `blk`: 256 consecutive vertices, or -- for an image of `cols` columns (cols % 32 == 0,
// rows % 8 == 0) -- a 32 x 8 pixel region whose warps are 8 x 4 patches.  Measured in the frame loop: the patch mapping pays because a warp's
// tighter queries walk the same grid cells in knn8_grid; warp-cooperative candidate lists on top of it were bit-exact but no faster.
__device__ __forceinline__ int patch_vertex(int blk, int tid, int cols)
{
    if (cols <= 0) return blk * 256 + tid;
    const int bpr = cols >> 5;
    const int bx = blk % bpr, by = blk / bpr;
    const int warp = tid >> 5, lane = tid & 31;
    return (by * 8 + (warp >> 2) * 4 + (lane >> 3)) * cols + bx * 32 + (warp & 3) * 8 + (lane & 7);
}

struct Quat { float w, x, y, z; };

// Quaternion::operator*, quaternion.hpp:191-199
__device__ __forceinline__ Quat qmul(const Quat a, const Quat b)
{
    Quat r;
    r.w = ((a.w * b.w) - (a.x * b.x) - (a.y * b.y) - (a.z * b.z));
    r.x = ((a.w * b.x) + (a.x * b.w) + (a.y * b.z) - (a.z * b.y));
    r.y = ((a.w * b.y) - (a.x * b.z) + (a.y * b.w) + (a.z * b.x));
    r.z = ((a.w * b.z) + (a.x * b.y) - (a.y * b.x) + (a.z * b.w));
    return r;
}
// Quaternion::normalize, quaternion.hpp:220-228: the scale 1.0/norm is a double, products narrowed to float
__device__ __forceinline__ Quat qnormalize(const Quat q)
{
    const float n = sqrtf((q.w * q.w) + (q.x * q.x) + (q.y * q.y) + (q.z * q.z));
    const double s = 1.0 / (double)n;
    Quat r;
    r.w = (float)(s * (double)q.w); r.x = (float)(s * (double)q.x); r.y = (float)(s * (double)q.y); r.z = (float)(s * (double)q.z);
    return r;
}
// DualQuaternion::getTranslation, dual_quaternion.hpp:120-125: 2 * translation_ * conj(normalised rotation_)
__device__ __forceinline__ Quat dq_translation(const Quat rot, const Quat dual)
{
    const Quat r = qnormalize(rot);
    const Quat conj = {r.w, -r.x, -r.y, -r.z};
    const Quat two = {2 * dual.w, 2 * dual.x, 2 * dual.y, 2 * dual.z};
    return qmul(two, conj);
}
// 0.5 * q with a double scalar (DualQuaternion ctor / encodeTranslation, dual_quaternion.hpp:59-63,82-85)
__device__ __forceinline__ Quat qhalf(const Quat q)
{
    Quat r;
    r.w = (float)(0.5 * (double)q.w); r.x = (float)(0.5 * (double)q.x); r.y = (float)(0.5 * (double)q.y); r.z = (float)(0.5 * (double)q.z);
    return r;
}
// Quaternion::rotate(Vec3f&), quaternion.hpp:124-130
__device__ __forceinline__ float3 qrotate(const Quat q, const float3 v)
{
    const Quat r = qnormalize(q);
    const float3 qv = make_float3(r.x, r.y, r.z);
    const float3 inner = add3(cross3(qv, v), scale3(v, r.w));
    const float3 c = cross3(scale3(qv, 2.f), inner);
    return make_float3(v.x + c.x, v.y + c.y, v.z + c.z);
}
// WarpField::weighting (warp_field.cpp:262-265): (float)exp((double)x), x = -d2 / (2 w^2) in float.  The generic double exp is ~60 instructions and
// was a large share of the warped-fusion kernel.  With the reference's node weight (3, i.e. sigma = 3 m) x
// lies in [-0.06, 0]; for x in [-0.5, 0] the value is formed as exp(-1/4) * P13(x + 1/4), a degree-13 Taylor polynomial in fused double
// arithmetic (truncation 2.4e-18, |r| <= 1/4): after the rounding to float it equals (float)exp((double)x) of a correctly rounded libm for
// EVERY float in the interval -- checked exhaustively, 1,056,964,609 values, by tests/test_weight_exp.py against glibc (the oracle's exp).
// Anything else (other node weights, NaN) takes the generic path.
// out of line: the generic exp is ~60 instructions, and kernels that weight eight neighbours per element would carry eight copies of it next to
// the polynomial -- the warped-fusion kernel turned out to be bound by instruction fetch
static __device__ __noinline__ float node_weighting_slow(float x) { return (float)exp((double)x); }

__device__ __forceinline__ float node_weighting(float d2, float node_w)
{
    const float x = -d2 / (2 * node_w * node_w);
    if (x >= -0.5f && x <= 0.f) {
        const double r = (double)x + 0.25;
        double p = 1.0 / 6227020800.0;
        p = __fma_rn(p, r, 1.0 / 479001600.0);
        p = __fma_rn(p, r, 1.0 / 39916800.0);
        p = __fma_rn(p, r, 1.0 / 3628800.0);
        p = __fma_rn(p, r, 1.0 / 362880.0);
        p = __fma_rn(p, r, 1.0 / 40320.0);
        p = __fma_rn(p, r, 1.0 / 5040.0);
        p = __fma_rn(p, r, 1.0 / 720.0);
        p = __fma_rn(p, r, 1.0 / 120.0);
        p = __fma_rn(p, r, 1.0 / 24.0);
        p = __fma_rn(p, r, 1.0 / 6.0);
        p = __fma_rn(p, r, 0.5);
        p = __fma_rn(p, r, 1.0);
        p = __fma_rn(p, r, 1.0);
        return (float)(0.77880078307140486825 * p);              // exp(-1/4)
    }
    return node_weighting_slow(x);
}

struct Dqb { Quat rot, dual; };

// WarpField::DQB (warp_field.cpp:203-217) from the 8 neighbours; weights8 (optional) receives the node weights
// kPrecomputedWeights: weights8 holds the weights on entry (re-use of a previous k-NN + weighting pass over the same
// query points); otherwise they are computed from the squared distances bd and written to weights8.
template <bool kPrecomputedWeights = false>
__device__ __forceinline__ Dqb dqb_blend(const float *__restrict__ nodes, const int (&bi)[8], const float (&bd)[8], float *weights8)
{
    Quat tsum = {0.f, 0.f, 0.f, 0.f}, rsum = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        float w = 0.f;
        if (bi[i] >= 0) {
            const float4 *n4 = reinterpret_cast<const float4 *>(nodes + (size_t)bi[i] * DF_NODE_STRIDE);
            const float4 a = __ldg(n4), b = __ldg(n4 + 1), c = __ldg(n4 + 2);   // (vx,vy,vz,rw) (rx,ry,rz,dw) (dx,dy,dz,weight)
            const Quat rot = {a.w, b.x, b.y, b.z};
            const Quat dual = {b.w, c.x, c.y, c.z};
            w = kPrecomputedWeights ? weights8[i] : node_weighting(bd[i], c.w);
            const Quat t = dq_translation(rot, dual);
            tsum.w = tsum.w + w * t.w; tsum.x = tsum.x + w * t.x; tsum.y = tsum.y + w * t.y; tsum.z = tsum.z + w * t.z;
            rsum.w = rsum.w + w * rot.w; rsum.x = rsum.x + w * rot.x; rsum.y = rsum.y + w * rot.y; rsum.z = rsum.z + w * rot.z;
        }
        if (!kPrecomputedWeights && weights8) weights8[i] = w;
    }
    Dqb r;
    r.rot = qnormalize(rsum);
    r.dual = qmul(qhalf(tsum), r.rot);     // DualQuaternion(translation, rotation) ctor
    return r;
}

// DualQuaternion::transform, dual_quaternion.hpp:204-210
__device__ __forceinline__ float3 dq_transform(const Dqb &d, const float3 v)
{
    const Quat t = dq_translation(d.rot, d.dual);
    const float3 r = qrotate(d.rot, v);
    return make_float3(r.x + t.x, r.y + t.y, r.z + t.z);
}

}  // namespace dfb
